"""Known-answer tests of the reference's ORDER BY operators, ported literally: every case of TopNExecTest and SortExecTest
(polardbx-executor/src/test/java/com/alibaba/polardbx/executor/operator/) whose columns are all integers.  The cases
that mix in a StringBlock (testIntegerMixString2Col..., testIntegerMixStringSensitive2Col...) need CHAR keys and are not
ported.

Each case: the MockExec chunks (per chunk, one list per column, None = NULL), the OrderByOption list as
(column, DESC?, NullDirection), the SpilledTopNExec topSize (None for SortExec), and the expected chunk.  `ordered` is the
third argument of the reference's assertExecResultByRow: SortExec results compare row by row, TopN results as multisets.
The null directions are carried although the executor never reads them: FIRST / UNSPECIFIED with DESC still puts NULLs
last (testInteger2ColTopN, testInteger2ColMemSort)."""

FIRST, LAST, UNSPECIFIED = "FIRST", "LAST", "UNSPECIFIED"
INT = 0  # DataTypes.IntegerType -> GSQL_T_INT32

_C4 = [
    [[None, 8, 9, 5], [9, 4, 3, 2]],
    [[3, 6, 1], [9, 4, 3]],
    [[None, 6, 15], [None, None, None]],
    [[3, 6, None], [96, 42, 33]],
]

TOPN_KATS = [
    dict(name="testIntegerTopN", types=[INT, INT],
         chunks=[[[None, 4, 5, 9], [3, 3, 4, 9]], [[1, 2, 3], [3, 4, 9]]],
         order=[(0, False, FIRST)], top=4,
         expect=[[None, 1, 2, 3], [3, 3, 4, 9]], ordered=False),
    dict(name="testInteger2ColTopN", types=[INT, INT],
         chunks=[[[None, 8, 9, 5], [9, 4, 3, 2]], [[3, 6, 1], [9, 4, 3]]],
         order=[(1, True, UNSPECIFIED), (0, True, UNSPECIFIED)], top=8,
         expect=[[3, None, 8, 6, 9, 1, 5], [9, 9, 4, 4, 3, 3, 2]], ordered=False),
    dict(name="testInteger2ColWithDiffDirectionsTopN", types=[INT, INT],
         chunks=[[[None, 8, 9, 5], [9, 4, 3, 2]], [[3, 6, 1], [9, 4, 3]]],
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], top=8,
         expect=[[None, 3, 6, 8, 1, 9, 5], [9, 9, 4, 4, 3, 3, 2]], ordered=False),
    dict(name="testInteger2ColWithDiffDirectionsAnd4InputsTopN", types=[INT, INT], chunks=_C4,
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], top=8,
         expect=[[3, 6, None, None, 3, 6, 8, 1], [96, 42, 33, 9, 9, 4, 4, 3]], ordered=False),
    dict(name="testInteger2ColWithDiffDirectionsAnd4InputsAndSkipTopN", types=[INT, INT], chunks=_C4,
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], top=7,
         expect=[[3, 6, None, None, 3, 6, 8], [96, 42, 33, 9, 9, 4, 4]], ordered=False),
    dict(name="testInteger2ColWithDiffDirectionsAnd4InputsAndSkipAndNullFetchTopN", types=[INT, INT], chunks=_C4,
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], top=90,
         expect=[[3, 6, None, None, 3, 6, 8, 1, 9, 5, None, 6, 15], [96, 42, 33, 9, 9, 4, 4, 3, 3, 2, None, None, None]],
         ordered=False),
]

SORT_KATS = [
    dict(name="testIntegerMemSort", types=[INT, INT],
         chunks=[[[None, 22, 5, 3], [3, 3, 4, 9]]],
         order=[(0, False, FIRST)], top=None,
         expect=[[None, 3, 5, 22], [3, 9, 4, 3]], ordered=True),
    dict(name="testIntegerWithNullMemSort", types=[INT, INT],
         chunks=[[[None, 22, 5, 3, -1], [3, 3, 4, 9, None]]],
         order=[(0, False, FIRST)], top=None,
         expect=[[None, -1, 3, 5, 22], [3, None, 9, 4, 3]], ordered=True),
    dict(name="testInteger2ColMemSort", types=[INT, INT],
         chunks=[[[None, 8, 5, 5], [9, 4, 3, 2]], [[3, 6, 1], [3, 3, 3]]],
         order=[(1, True, UNSPECIFIED), (0, True, UNSPECIFIED)], top=None,
         expect=[[None, 8, 6, 5, 3, 1, 5], [9, 4, 3, 3, 3, 3, 2]], ordered=True),
    dict(name="testInteger2ColWithDiffDirectionsMemSort", types=[INT, INT],
         chunks=[[[None, 8, 5, 5], [9, 9, 3, 2]], [[3, 6, 1], [3, 3, 3]]],
         order=[(1, True, UNSPECIFIED), (0, False, UNSPECIFIED)], top=None,
         expect=[[None, 8, 1, 3, 5, 6, 5], [9, 9, 3, 3, 3, 3, 2]], ordered=True),
    dict(name="testInteger2ColWithDiffDirectionsAnd4InputsMergeSort", types=[INT, INT], chunks=_C4,
         order=[(1, False, UNSPECIFIED), (0, True, UNSPECIFIED)], top=None,
         expect=[[15, 6, None, 5, 9, 1, 8, 6, 3, None, None, 6, 3], [None, None, None, 2, 3, 3, 4, 4, 9, 9, 33, 42, 96]],
         ordered=True),
]

ALL_KATS = TOPN_KATS + SORT_KATS
