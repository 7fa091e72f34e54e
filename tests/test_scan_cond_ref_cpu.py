"""Pins tests/scan_cond_ref.py, the restatement of the reference's CASE, COALESCE, IN, BETWEEN and DATE-comparison
classes, with hand-worked values written out as literals (file:line citations in scan_cond_ref's docstring); and checks
that the programs the GPU runs (ops 32..36) compute those classes."""
import numpy as np

from tests import scan_cond_ref as Q
from tests import scan_ref as R

NULL = None
C0, C1, C2 = (R.OP_COL, 0, 0), (R.OP_COL, 1, 0), (R.OP_COL, 2, 0)


def _col(vals, dtype=np.int64):
    nl = np.array([v is None for v in vals], bool)
    return np.array([0 if v is None else v for v in vals], dtype=dtype), nl


def _list(c):
    v, nl = c
    return [None if n else x for x, n in zip(np.asarray(v).tolist(), np.asarray(nl).tolist())]


def test_case_first_true_condition_wins_and_null_conditions_are_not_taken():
    # CaseVectorizedExpression.java:83-103: each when narrows the rows still open; conditionalEval keeps TRUE rows only
    w1 = _col([1, 0, NULL, 1, NULL, 0])
    w2 = _col([1, 1, 1, NULL, NULL, 0])
    t1, t2, e = _col([10] * 6), _col([20, 20, NULL, 20, 20, 20]), _col([30, 30, 30, 30, 30, NULL])
    assert _list(Q.ref_case([w1, w2], [t1, t2], e)) == [10, 20, NULL, 10, 30, NULL]
    # a missing ELSE (Calcite's NULL literal): rows no condition takes are NULL
    assert _list(Q.ref_case([w1, w2], [t1, t2], None)) == [10, 20, NULL, 10, NULL, NULL]
    # a condition's value under its NULL flag is never read
    dirty = (np.array([1, 1], np.int64), np.array([True, False]))
    assert _list(Q.ref_case([dirty], [_col([7, 7])], _col([8, 8]))) == [8, 7]


def test_coalesce_takes_the_first_non_null():
    a, b, c = _col([1, NULL, NULL, NULL]), _col([2, 5, NULL, NULL]), _col([3, 6, 9, NULL])
    assert _list(Q.ref_coalesce([a, b, c])) == [1, 5, 9, NULL]
    assert _list(Q.ref_coalesce([a])) == [1, NULL, NULL, NULL]


def test_in_compares_the_value_under_a_null_flag_and_a_null_constant_nulls_every_row():
    # AbstractInLongColLongConstVectorizedExpression.java:99-111: anyMatch(value), no NULL merge; appendNull stores 0
    x = _col([0, 5, NULL, 7, -(1 << 63)])
    assert _list(Q.ref_in(x, [0, 5])) == [1, 1, 1, 0, 0]                      # NULL IN (0, 5) is TRUE
    assert _list(Q.ref_in(x, [7])) == [0, 0, 0, 1, 0]                         # NULL IN (7) is FALSE, not NULL
    assert _list(Q.ref_in(x, [-(1 << 63), 3])) == [0, 0, 0, 0, 1]
    # lines 90-97: one NULL constant -> every row NULL, whatever matches
    assert _list(Q.ref_in(x, [0, NULL, 5])) == [NULL] * 5
    # an INT column compares widened to long (AbstractInIntegerColLongConst... anyMatch(int))
    assert _list(Q.ref_in(_col([5, -1], np.int32), [(1 << 32) + 5, -1])) == [0, 1]


def test_between_has_the_in_null_rules():
    # BetweenLongColLongConstLongConstVectorizedExpression.java:78-85 and 93-96
    x = _col([1, 2, 3, 4, NULL])
    assert _list(Q.ref_between(x, 2, 3)) == [0, 1, 1, 0, 0]
    assert _list(Q.ref_between(x, -1, 1)) == [1, 0, 0, 0, 1]                  # NULL BETWEEN -1 AND 1 is TRUE
    assert _list(Q.ref_between(x, 3, 2)) == [0] * 5
    assert _list(Q.ref_between(x, NULL, 3)) == [NULL] * 5
    assert _list(Q.ref_between(x, 1, NULL)) == [NULL] * 5


def test_date_constant_is_the_packed_long_and_rows_compare_packed():
    # TimeStorage.writeDate: ((y * 13 + m) << 5 | d) << 41
    assert Q.write_date(1995, 3, 15) == ((1995 * 13 + 3) << 5 | 15) << 41 == 1825257471829082112
    assert Q.pack_days(np.array([9204]))[0] == Q.write_date(1995, 3, 15)        # day 9204 is 1995-03-15
    assert Q.pack_days(np.array([0, 59, 365 * 3 + 59]))[:2].tolist() == [Q.write_date(1970, 1, 1), Q.write_date(1970, 3, 1)]
    assert Q.pack_days(np.array([365 * 2 + 59]))[0] == Q.write_date(1972, 2, 29)  # a leap day
    days = np.arange(8035, 8035 + 2557)                                          # 1992-01-01 .. 1998-12-31
    p = Q.pack_days(days)
    assert (np.diff(p) > 0).all()                                                # packing keeps the order of dates
    col = _col([Q.write_date(1995, 3, 14), Q.write_date(1995, 3, 15), NULL, Q.write_date(1996, 1, 1)])
    k = Q.write_date(1995, 3, 15)
    assert _list(Q.ref_date_cmp(col, R.OP_LT, k)) == [1, 0, NULL, 0]           # the column's NULL is merged
    assert _list(Q.ref_date_cmp(col, R.OP_GE, k)) == [0, 1, NULL, 1]
    assert _list(Q.ref_date_cmp(col, R.OP_NE, NULL)) == [NULL] * 4             # a NULL literal: every row NULL


def test_programs_compute_the_reference_classes():
    """The forms the translator emits: CASE right to left, a missing ELSE as CONST_NULL, COALESCE folded left, IN / BETWEEN
    over a column, a NULL constant in IN / BETWEEN as CONST_NULL, a DATE comparison as COL <cmp> CONST_I64."""
    a, b, c = _col([1, 0, NULL, 1, 0]), _col([0, 1, 1, NULL, 0]), _col([4, NULL, 6, 7, 8])
    cols = [a, b, c]
    case = [C2, C0, (R.OP_CONST_I64, 0, 10), Q.OP_CASE_WHEN, C1, (R.OP_CONST_I64, 0, 20), Q.OP_CASE_WHEN]
    case = [i if isinstance(i, tuple) else (i, 0, 0) for i in case]
    # CASE WHEN b THEN 20 WHEN a THEN 10 ELSE c END
    assert _list(Q.evaluate(case, cols)) == _list(Q.ref_case([b, a], [_col([20] * 5), _col([10] * 5)], c)) == [10, 20, 20, 10, 8]
    no_else = [(Q.OP_CONST_NULL, R.T_INT64, 0), C1, (R.OP_CONST_I64, 0, 20), (Q.OP_CASE_WHEN, 0, 0)]
    assert _list(Q.evaluate(no_else, cols)) == [NULL, 20, 20, NULL, NULL]
    coal = [C2, C0, (Q.OP_COALESCE, 0, 0), C1, (Q.OP_COALESCE, 0, 0)]
    assert _list(Q.evaluate(coal, cols)) == _list(Q.ref_coalesce([c, a, b])) == [4, 0, 6, 7, 8]
    pool = [7, 4, 0, 6]
    assert _list(Q.evaluate([C2, (Q.OP_IN, 0, 3)], cols, pool)) == _list(Q.ref_in(c, [7, 4, 0])) == [1, 1, 0, 1, 0]
    assert _list(Q.evaluate([C2, (Q.OP_BETWEEN, 2, 2)], cols, pool)) == _list(Q.ref_between(c, 0, 6)) == [1, 1, 1, 0, 0]
    assert _list(Q.evaluate([(Q.OP_CONST_NULL, R.T_INT64, 0)], cols)) == _list(Q.ref_in(c, [1, NULL])) == [NULL] * 5
    # the constants travel in the instruction as api.E builds it, too
    assert _list(Q.evaluate([C2, (Q.OP_IN, 0, (0, 4, 7))], cols)) == [1, 1, 0, 1, 0]
    # IN over a computed operand reads 0 where the operand is NULL (the GPU's rule; the translator never sends it)
    assert _list(Q.evaluate([C2, (R.OP_CONST_I64, 0, 1), (R.OP_ADD, 0, 0), (Q.OP_IN, 0, (0, 5))], cols)) == [1, 1, 0, 0, 0]


def test_checker_verdicts():
    t = [R.T_INT32, R.T_INT64, R.T_FP64]
    I, D = (R.OP_CONST_I64, 0, 1), (R.OP_CONST_F64, 0, 1.0)
    cw, co = (Q.OP_CASE_WHEN, 0, 0), (Q.OP_COALESCE, 0, 0)
    ok = [([C1, C0, I, cw], R.T_INT64), ([D, C0, C2, cw], R.T_FP64), ([(Q.OP_CONST_NULL, R.T_FP64, 0)], R.T_FP64),
          ([C0, I, co], R.T_INT64), ([C0, (Q.OP_IN, 0, 1)], R.T_INT64), ([C1, (Q.OP_BETWEEN, 0, 0)], R.T_INT64),
          ([C0, C1, (R.OP_ADD, 0, 0), (Q.OP_IN, 0, 2)], R.T_INT64)]
    for ins, want in ok:
        assert Q.check(ins, t, 2) == (want, None), ins
    bad = [([C1, D, I, cw], "condition is a double"), ([C1, C0, D, cw], "branch types"), ([C0, I], "leaves 2 values"),
           ([C0, D, co], "branch types"), ([C2, (Q.OP_IN, 0, 1)], "set over a double"), ([C0, (Q.OP_IN, 0, 0)], "list length"),
           ([C0, (Q.OP_IN, 0, 257)], "list length"), ([C0, (Q.OP_IN, 1, 2)], "pool range"), ([C0, (Q.OP_IN, -1, 1)], "pool range"),
           ([C0, (Q.OP_BETWEEN, 1, 0)], "pool range"), ([(Q.OP_CONST_NULL, R.T_INT32, 0)], "null type"), ([C0, C0, cw], "underflow"),
           ([C0, (37, 0, 0)], "unknown op"), ([C0, (31, 0, 0)], "unknown op"), ([I, I, I, I, (Q.OP_CONST_NULL, R.T_INT64, 0)], "depth")]
    for ins, why in bad:
        assert Q.check(ins, t, 2) == (None, why), ins
    # the pool holds at most 1024 entries over all programs' lists
    big = [C0, (Q.OP_IN, 0, 256)]
    assert Q.check_scan(t, [big] * 4, npool=256)[0] == [R.T_INT64] * 4
    assert Q.check_scan(t, [big] * 4, big, npool=256) == (None, "pool size")
    assert Q.check_scan(t, [[C0]], npool=1025) == (None, "pool")


def test_checker_agrees_with_scan_ref_on_old_programs():
    rng = np.random.default_rng(3)
    t = [R.T_INT32, R.T_INT64, R.T_FP64]
    ops = [R.OP_COL, R.OP_CONST_I64, R.OP_CONST_F64] * 3 + list(R.ARITH + R.COMPARE + R.LOGIC + R.UNARY)
    for _ in range(3000):
        ins = [(int(ops[rng.integers(len(ops))]), int(rng.integers(0, 3)), 1) for _ in range(int(rng.integers(1, 8)))]
        assert (Q.check(ins, t)[0]) == R.check(ins, t)[0], ins
