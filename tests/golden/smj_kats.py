"""Known-answer tests of the reference's SortMergeJoinExec, ported from SortMergeJoinExecTest
(polardbx-executor/src/test/java/com/alibaba/polardbx/executor/operator/SortMergeJoinExecTest.java): all 23 cases.

String columns become INT codes: `encode` maps each distinct string of a case to an integer in the strings' order (NULL
stays NULL).  That keeps every comparison the cases make.  Only testInnerJoin_MultiKey has a string key, and it holds only
"a", "b", "c" and NULL; everywhere else strings are payloads, compared at most for equality by the WithCondition cases.
The data below keeps the strings as the reference writes them.

Each case: the outer and inner MockExec chunks (per chunk, one list per column, None = NULL), the column types, the join
type, maxOneRow, the keys as (outerIndex, innerIndex) with unified type INT, every key ascending (mockSortMergeJoinExec),
the anti-join operands as outer column indexes (InputRefExpression) or None, the other condition as
("ne", joinRowColumn, value) meaning !Objects.equals(row.getObject(column), value) or None, and the expected chunk
(None: "more than 1 row" is raised).  assertExecResults compares the rows as multisets; the restatement's row order is
checked separately."""

INT, STR = "int", "str"
INNER, LEFT, RIGHT, SEMI, ANTI = "INNER", "LEFT", "RIGHT", "SEMI", "ANTI"

_OUTER_A = [[[0, 1, 2, 3], [None, 1, 1, 2]], [[4, 5, 6, 7, 8], [3, 4, 5, 6, 7]]]
_OUTER_A9 = [[[0, 1, 2, 3], [None, 1, 1, 2]], [[4, 5, 6, 7, 8], [3, 4, 5, 6, 9]]]
_INNER_A = [[[1, 1, 2, 2], ["a", "b", "c", None]], [[4, 5, 6, 7], ["d", "e", "f", None]]]
_INNER_A_NULL = [[[None, 1, 1, 2, 2], ["!", "a", "b", "c", None]], [[4, 5, 6, 7], ["d", "e", "f", None]]]
_INNER_SEMI = [[[None, 1, 1, 2, 2]], [[4, 5, 6, 7]]]
_OUTER_B = [[[7, 0, 5, 1], [None, 3, 3, 4]], [[4, 3, 6, 2], [5, 7, 8, 9]]]
_INNER_B = [[[1, 2, 3, 4]], [[3, 4, 5, 6]]]
_OUTER_C = [[[7, 5, 0, 1], [1, 3, 3, 4]], [[4, 3, 6, 2], [5, 7, 8, 9]]]
_INNER_C = [[["a", "b", "c", None], [1, 2, 3, 4]], [["d", "e", "f", None], [5, 6, 7, 8]]]
_INNER_C_DUP = [[["a", "b", "c", None], [1, 2, 3, 4]], [["d", "e", "f", None], [4, 5, 6, 7]]]

SMJ_KATS = [
    dict(name="testInnerJoin_Simple", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT, STR], inner=_INNER_A,
         join=INNER, single=False, keys=[(1, 0)], anti=None, cond=None,
         expect=[[1, 1, 2, 2, 3, 3, 5, 6, 7, 8], [1, 1, 1, 1, 2, 2, 4, 5, 6, 7], [1, 1, 1, 1, 2, 2, 4, 5, 6, 7],
                 ["a", "b", "a", "b", "c", None, "d", "e", "f", None]]),
    dict(name="testInnerJoin_EmptyInnerSide", outer_types=[INT, INT],
         outer=[[[0, 1, 2, 3], [1, 1, 1, 2]], [[4, 5, 6, 7, 8], [3, 4, 5, 6, 7]]], inner_types=[INT, STR], inner=[],
         join=INNER, single=False, keys=[(1, 0)], anti=None, cond=None, expect=[[], [], [], []]),
    dict(name="testInnerJoin_EmptyOuterSide", outer_types=[INT, INT], outer=[], inner_types=[INT, STR], inner=_INNER_A,
         join=INNER, single=False, keys=[(1, 0)], anti=None, cond=None, expect=[[], [], [], []]),
    dict(name="testInnerJoin_EmptyBothSides", outer_types=[INT, INT], outer=[], inner_types=[INT, STR], inner=[],
         join=INNER, single=False, keys=[(1, 0)], anti=None, cond=None, expect=[[], [], [], []]),
    dict(name="testInnerJoin_MultiKey", outer_types=[INT, INT, STR],
         outer=[[[-1, 0, 1, 2, 3], [0, 1, 1, 2, 2], [None, "a", "b", "a", "b"]],
                [[5, 6, 7, 8], [3, 3, 4, 4], ["a", "b", "a", "b"]]],
         inner_types=[INT, STR, STR],
         inner=[[[None, 1, 1, 2], ["b", "a", "a", "a"], ["H", "A", "E", "B"]],
                [[2, 3, 3, 4], ["b", "a", "c", None], ["F", "C", "G", "D"]]],
         join=INNER, single=False, keys=[(1, 0), (2, 1)], anti=None, cond=None,
         expect=[[0, 0, 2, 3, 5], [1, 1, 2, 2, 3], ["a", "a", "a", "b", "a"], [1, 1, 2, 2, 3], ["a", "a", "a", "b", "a"],
                 ["A", "E", "B", "F", "C"]]),
    dict(name="testLeftOuterJoin_Simple", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT, STR], inner=_INNER_A_NULL,
         join=LEFT, single=False, keys=[(1, 0)], anti=None, cond=None,
         expect=[[0, 1, 1, 2, 2, 3, 3, 4, 5, 6, 7, 8], [None, 1, 1, 1, 1, 2, 2, 3, 4, 5, 6, 7],
                 [None, 1, 1, 1, 1, 2, 2, None, 4, 5, 6, 7], [None, "a", "b", "a", "b", "c", None, None, "d", "e", "f", None]]),
    dict(name="testLeftOuterJoin_WithCondition", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT, STR],
         inner=_INNER_A_NULL, join=LEFT, single=False, keys=[(1, 0)], anti=None, cond=("ne", 3, "d"),
         expect=[[0, 1, 1, 2, 2, 3, 3, 4, 5, 6, 7, 8], [None, 1, 1, 1, 1, 2, 2, 3, 4, 5, 6, 7],
                 [None, 1, 1, 1, 1, 2, 2, None, None, 5, 6, 7], [None, "a", "b", "a", "b", "c", None, None, None, "e", "f", None]]),
    # the reference's expected chunk gives its last two blocks ten NULLs for nine rows; the nine rows are what it compares
    dict(name="testLeftOuterJoin_InnerEmpty", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT, STR], inner=[],
         join=LEFT, single=False, keys=[(1, 0)], anti=None, cond=None,
         expect=[[0, 1, 2, 3, 4, 5, 6, 7, 8], [None, 1, 1, 2, 3, 4, 5, 6, 7], [None] * 9, [None] * 9]),
    dict(name="testRightOuterJoin_Simple", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT, STR], inner=_INNER_A,
         join=RIGHT, single=False, keys=[(1, 0)], anti=None, cond=None,
         expect=[[None, 1, 1, 1, 1, 2, 2, None, 4, 5, 6, 7], [None, "a", "b", "a", "b", "c", None, None, "d", "e", "f", None],
                 [0, 1, 1, 2, 2, 3, 3, 4, 5, 6, 7, 8], [None, 1, 1, 1, 1, 2, 2, 3, 4, 5, 6, 7]]),
    dict(name="testRightOuterJoin_InnerEmpty", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT, STR], inner=[],
         join=RIGHT, single=False, keys=[(1, 0)], anti=None, cond=None,
         expect=[[None] * 9, [None] * 9, [0, 1, 2, 3, 4, 5, 6, 7, 8], [None, 1, 1, 2, 3, 4, 5, 6, 7]]),
    dict(name="testSemiJoin_Simple", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT], inner=_INNER_SEMI,
         join=SEMI, single=False, keys=[(1, 0)], anti=None, cond=None,
         expect=[[1, 2, 3, 5, 6, 7, 8], [1, 1, 2, 4, 5, 6, 7]]),
    dict(name="testSemiJoin_InnerEmpty", outer_types=[INT, INT], outer=_OUTER_A, inner_types=[INT], inner=[],
         join=SEMI, single=False, keys=[(1, 0)], anti=None, cond=None, expect=[[], []]),
    dict(name="testAntiJoin_NotExists", outer_types=[INT, INT], outer=_OUTER_B, inner_types=[INT], inner=_INNER_B,
         join=ANTI, single=False, keys=[(1, 0)], anti=None, cond=None, expect=[[7, 3, 6, 2], [None, 7, 8, 9]]),
    dict(name="testAntiJoin_NotIn", outer_types=[INT, INT], outer=_OUTER_B, inner_types=[INT], inner=_INNER_B,
         join=ANTI, single=False, keys=[(1, 0)], anti=[1], cond=None, expect=[[3, 6, 2], [7, 8, 9]]),
    dict(name="testAntiJoin_NotIn_InnerEmpty", outer_types=[INT, INT], outer=[[[7, 0, 5, 1], [None, None, 3, 4]]],
         inner_types=[INT], inner=[], join=ANTI, single=False, keys=[(1, 0)], anti=[1], cond=None,
         expect=[[7, 0, 5, 1], [None, None, 3, 4]]),
    dict(name="testAntiJoin_NotIn_InnerContainsNull", outer_types=[INT, INT], outer=_OUTER_B, inner_types=[INT],
         inner=[[[None, 2, 3, 4]], [[3, 4, 5, 6]]], join=ANTI, single=False, keys=[(1, 0)], anti=[1], cond=None,
         expect=[[], []]),
    dict(name="testAntiJoin_InnerEmpty", outer_types=[INT, INT], outer=_OUTER_A9, inner_types=[INT], inner=[],
         join=ANTI, single=False, keys=[(1, 0)], anti=None, cond=None,
         expect=[[0, 1, 2, 3, 4, 5, 6, 7, 8], [None, 1, 1, 2, 3, 4, 5, 6, 9]]),
    dict(name="testAntiJoin_WithCondition", outer_types=[INT, INT], outer=_OUTER_A9, inner_types=[INT], inner=_INNER_SEMI,
         join=ANTI, single=False, keys=[(1, 0)], anti=None, cond=("ne", 2, 4), expect=[[0, 4, 5, 8], [None, 3, 4, 9]]),
    dict(name="testInnerSingleJoin", outer_types=[INT, INT], outer=_OUTER_C, inner_types=[STR, INT], inner=_INNER_C,
         join=INNER, single=True, keys=[(1, 1)], anti=None, cond=None,
         expect=[[7, 5, 0, 1, 4, 3, 6], [1, 3, 3, 4, 5, 7, 8], ["a", "c", "c", None, "d", "f", None]]),
    dict(name="testInnerSingleJoin_withError", outer_types=[INT, INT], outer=_OUTER_C, inner_types=[STR, INT],
         inner=_INNER_C_DUP, join=INNER, single=True, keys=[(1, 1)], anti=None, cond=None, expect=None),
    dict(name="testLeftSingleJoin", outer_types=[INT, INT], outer=_OUTER_C, inner_types=[STR, INT], inner=_INNER_C,
         join=LEFT, single=True, keys=[(1, 1)], anti=None, cond=None,
         expect=[[7, 5, 0, 1, 4, 3, 6, 2], [1, 3, 3, 4, 5, 7, 8, 9], ["a", "c", "c", None, "d", "f", None, None]]),
    dict(name="testLeftSingleJoin_WithCondition", outer_types=[INT, INT], outer=_OUTER_C, inner_types=[STR, INT],
         inner=_INNER_C, join=LEFT, single=True, keys=[(1, 1)], anti=None, cond=("ne", 2, "d"),
         expect=[[7, 5, 0, 1, 4, 3, 6, 2], [1, 3, 3, 4, 5, 7, 8, 9], ["a", "c", "c", None, None, "f", None, None]]),
    dict(name="testLeftSingleJoin_withError", outer_types=[INT, INT], outer=_OUTER_C, inner_types=[STR, INT],
         inner=_INNER_C_DUP, join=LEFT, single=True, keys=[(1, 1)], anti=None, cond=None, expect=None),
]


def encode(case):
    """The case with every string replaced by its code: the rank of the string among the case's distinct strings."""
    strings = set()

    def collect(v):
        if isinstance(v, str):
            strings.add(v)

    for side in ("outer", "inner"):
        for ch in case[side]:
            for col in ch:
                for v in col:
                    collect(v)
    for col in case["expect"] or []:
        for v in col:
            collect(v)
    if case["cond"]:
        collect(case["cond"][2])
    code = {s: i for i, s in enumerate(sorted(strings))}
    enc = lambda v: code[v] if isinstance(v, str) else v
    out = dict(case)
    for side in ("outer", "inner"):
        out[side] = [[[enc(v) for v in col] for col in ch] for ch in case[side]]
        out[side + "_types"] = [INT for _ in case[side + "_types"]]
    out["expect"] = None if case["expect"] is None else [[enc(v) for v in col] for col in case["expect"]]
    if case["cond"]:
        out["cond"] = (case["cond"][0], case["cond"][1], enc(case["cond"][2]))
    return out
