"""Known-answer tests of the reference's MergeSortExec, ported literally: every case of MergeSortExecTest
(polardbx-executor/src/test/java/com/alibaba/polardbx/executor/operator/MergeSortExecTest.java) whose columns are all
integers.  testIntegerMixString2ColWithDiffDirectionsAnd4InputsMergeSort mixes in a StringBlock (CHAR keys) and is not
ported.

Each case: the MockExec inputs, kept separate (per input, its chunks; per chunk, one list per column, None = NULL), the
OrderByOption list as (column, DESC?, NullDirection), the MergeSortExec offset and limit, and the expected chunk.  The
reference compares results row by row (assertExecResults)."""

FIRST, LAST, UNSPECIFIED = "FIRST", "LAST", "UNSPECIFIED"
INT = 0  # DataTypes.IntegerType -> GSQL_T_INT32

_IN2 = [
    [[[None, 8, 9, 5], [9, 4, 3, 2]]],
    [[[3, 6, 1], [9, 4, 3]]],
]
_IN4 = _IN2 + [
    [[[None, 6, 15], [None, None, None]]],
    [[[3, 6, None], [96, 42, 33]]],
]

MERGE_KATS = [
    dict(name="testIntegerMergeSort", types=[INT, INT],
         inputs=[[[[None, 4, 5, 9], [3, 3, 4, 9]]], [[[1, 2, 3], [3, 4, 9]]]],
         order=[(0, False, FIRST)], offset=0, limit=4,
         expect=[[None, 1, 2, 3], [3, 3, 4, 9]]),
    dict(name="testIntegerNegativeMergeSort", types=[INT, INT],
         inputs=[[[[None, -1, 4, 5, 9], [3, None, 3, 4, 9]]], [[[1, 2, 3], [3, 4, 9]]]],
         order=[(0, False, FIRST)], offset=0, limit=4,
         expect=[[None, -1, 1, 2], [3, None, 3, 4]]),
    dict(name="testInteger2ColMergeSort", types=[INT, INT], inputs=_IN2,
         order=[(1, True, UNSPECIFIED), (0, True, UNSPECIFIED)], offset=0, limit=8,
         expect=[[3, None, 8, 6, 9, 1, 5], [9, 9, 4, 4, 3, 3, 2]]),
    dict(name="testInteger2ColWithDiffDirectionsMergeSort", types=[INT, INT], inputs=_IN2,
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], offset=0, limit=8,
         expect=[[None, 3, 6, 8, 1, 9, 5], [9, 9, 4, 4, 3, 3, 2]]),
    dict(name="testInteger2ColWithDiffDirectionsAnd4InputsMergeSort", types=[INT, INT], inputs=_IN4,
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], offset=0, limit=8,
         expect=[[3, 6, None, None, 3, 6, 8, 1], [96, 42, 33, 9, 9, 4, 4, 3]]),
    dict(name="testInteger2ColWithDiffDirectionsAnd4InputsAndSkipMergeSort", types=[INT, INT], inputs=_IN4,
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], offset=4, limit=3,
         expect=[[3, 6, 8], [9, 4, 4]]),
]
