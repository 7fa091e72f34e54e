"""Known-answer test of the reference's ExpandExec, ported literally from ExpandExecTest
(polardbx-executor/src/test/java/com/alibaba/polardbx/executor/operator/ExpandExecTest.java): one chunk of two INT
columns, two projections of one output column each (InputRef 0, then InputRef 1), and the expected output rows in order.

Each case: the MockExec chunks (per chunk, one list per column), the input types, the output types, the projections
(per projection one item per output column: an int = InputRefExpression(i)) and the expected rows of the single output
column, compared as a multiset (execForSmpMode with order = true still compares the rows the operator returned)."""

INT = "int"

EXPAND_KATS = [
    dict(name="test", types=[INT, INT], chunks=[[[1, 2, 3, 4], [5, 6, 7, 8]]], out_types=[INT], projections=[[0], [1]],
         expect=[[1, 2, 3, 4, 5, 6, 7, 8]]),
]
