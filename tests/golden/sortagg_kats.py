"""Known-answer tests of the reference's SortAggExec, ported literally from SortAggExecTest
(polardbx-executor/src/test/java/com/alibaba/polardbx/executor/operator/SortAggExecTest.java): every case whose columns
are integers or doubles.  testLargeNumerberBigDecimalSum and testBigDecimalNullAvg aggregate DECIMAL values and are not
ported (DECIMAL stays on the stock operator).  testDoubleNullAvg's value column is taken as DOUBLE, as
reference_kats.py ports the hash aggregation's AVG cases: AVG over INT is a DECIMAL division the GPU path refuses.

Each case: the MockExec chunks (per chunk, one list per column, None = NULL; a chunk of None is the reference's
withChunk(null)), the column types, the group columns, the aggregate calls as (kind, columns) and the expected chunk,
compared row by row in order (assertExecResultByRow with order = false compares the row lists as given)."""

INT, DOUBLE = "int", "double"

_NULL_VALUES = [[[0, 0, 1, 1], [None, None, None, None]], [[2, 2, 3, 3], [None, None, None, None]]]

SORTAGG_KATS = [
    dict(name="testInputIsNull", types=[INT, INT], chunks=[None, None], groups=[0], aggs=[("COUNT", [1])],
         expect=[[], []]),
    dict(name="testSimpleCount", types=[INT, INT],
         chunks=[[[0, 0, 1, 1], [3, 4, 9, 7]], [[2, 2, 3, 3], [5, 3, 8, 1]]], groups=[0], aggs=[("COUNT", [1])],
         expect=[[0, 1, 2, 3], [2, 2, 2, 2]]),
    dict(name="testSimpleSum", types=[INT, INT],
         chunks=[[[0, 0, 1, 1], [3, 5, 4, 3]], [[2, 2, 3, 3], [9, 8, 1, 7]]], groups=[0], aggs=[("SUM", [1])],
         expect=[[0, 1, 2, 3], [8, 7, 17, 8]]),
    dict(name="testDoubleNullAvg", types=[INT, DOUBLE], chunks=_NULL_VALUES, groups=[0], aggs=[("AVG", [1])],
         expect=[[0, 1, 2, 3], [None, None, None, None]]),
    dict(name="testNullSum", types=[INT, INT], chunks=_NULL_VALUES, groups=[0], aggs=[("SUM", [1])],
         expect=[[0, 1, 2, 3], [None, None, None, None]]),
    dict(name="testNullCount", types=[INT, INT], chunks=_NULL_VALUES, groups=[0], aggs=[("COUNT", [1])],
         expect=[[0, 1, 2, 3], [0, 0, 0, 0]]),
]
