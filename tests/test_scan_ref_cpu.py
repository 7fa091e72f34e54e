"""Pins tests/scan_ref.py, the numpy restatement of the reference's expression semantics that the GPU scan tests compare
against, with hand-worked values written out as literals; and checks by text that GpuExpression.java hands the GPU only
the divisions and casts whose reference semantics gsql_scan implements."""
import itertools
import math
import os
import re
import struct

import numpy as np

from tests import scan_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIN, MAX = R.INT64_MIN, R.INT64_MAX
NAN, INF = float("nan"), float("inf")
NULL = None


def _col(vals, dtype):
    """Python list with None -> (values, nulls)."""
    nl = np.array([v is None for v in vals], bool)
    return np.array([0 if v is None else v for v in vals], dtype=dtype), nl


def _run(ins, *cols):
    """-> the result as a Python list, None for NULL; doubles as (sign-aware) floats."""
    v, nl = R.evaluate(ins, list(cols))
    return [None if n else x for x, n in zip(v.tolist(), nl.tolist())]


def _same(got, exp):
    """List equality that tells -0.0 from 0.0 and lets NaN equal NaN."""
    assert len(got) == len(exp), (got, exp)
    for g, e in zip(got, exp):
        if isinstance(e, float):
            assert isinstance(g, float) and (struct.pack("<d", g) == struct.pack("<d", e) or (math.isnan(g) and math.isnan(e))), (got, exp)
        else:
            assert g == e and type(g) is type(e), (got, exp)


C0, C1 = (R.OP_COL, 0, 0), (R.OP_COL, 1, 0)


def test_cast_to_bigint_rounds_half_to_even_and_saturates():
    x = _col([0.5, 1.5, 2.5, -0.5, -2.5, 2.7, -2.7, 9.3e18, -9.3e18, INF, -INF, NAN, 9007199254740993.0, 9223372036854774784.0,
              -9223372036854775808.0, 0.49999999999999994, NULL], np.float64)
    _same(_run([C0, (R.OP_CAST_I64, 0, 0)], x),
          [0, 2, 2, 0, -2, 3, -3, MAX, MIN, MAX, MIN, 0, 9007199254740992, 9223372036854774784, MIN, 0, NULL])
    i = _col([MIN, MAX, -1, NULL], np.int64)
    _same(_run([C0, (R.OP_CAST_I64, 0, 0)], i), [MIN, MAX, -1, NULL])                       # of a long: the identity
    # (double) long rounds to nearest even: 2^53 + 1 -> 2^53, 2^53 + 3 -> 2^53 + 4, MAX -> 2^63
    _same(_run([C0, (R.OP_CAST_F64, 0, 0)], _col([(1 << 53) + 1, (1 << 53) + 3, MAX, MIN, NULL], np.int64)),
          [9007199254740992.0, 9007199254740996.0, 9223372036854775808.0, -9223372036854775808.0, NULL])


def test_division_by_zero_is_null_and_by_nan_is_not():
    div = [C0, C1, (R.OP_DIV, 0, 0)]
    x = _col([1.0, 1.0, 1.0, 0.0, 1.0, -1.0, NULL, 6.0], np.float64)
    y = _col([0.0, -0.0, NAN, 0.0, INF, 5e-324, 2.0, NULL], np.float64)
    _same(_run(div, x, y), [NULL, NULL, NAN, NULL, 0.0, -INF, NULL, NULL])
    # a long divisor is compared after (double): 0 is NULL; the quotient is always a double
    _same(_run(div, _col([7, 0, MIN, 1], np.int64), _col([0, 0, -1, MAX], np.int64)),
          [NULL, NULL, 9223372036854775808.0, 1.0 / 9223372036854775808.0])
    _same(_run([C0, (R.OP_CONST_I64, 0, 0), (R.OP_DIV, 0, 0)], _col([3, NULL], np.int32)), [NULL, NULL])     # a zero constant: the whole column
    _same(_run([C0, (R.OP_CONST_F64, 0, -0.0), (R.OP_DIV, 0, 0)], _col([3.5], np.float64)), [NULL])
    _same(_run([(R.OP_CONST_I64, 0, 1), C0, (R.OP_DIV, 0, 0)], _col([4, 0, -0.0, NAN], np.float64)), [0.25, NULL, NULL, NAN])
    assert R.check(div, [R.T_INT32, R.T_INT32]) == (R.T_FP64, None)


def test_three_valued_logic_tables():
    a = _col([1, 1, 1, 0, 0, 0, NULL, NULL, NULL], np.int64)
    b = _col([1, 0, NULL, 1, 0, NULL, 1, 0, NULL], np.int64)
    _same(_run([C0, C1, (R.OP_AND, 0, 0)], a, b), [1, 0, NULL, 0, 0, 0, NULL, 0, NULL])
    _same(_run([C0, C1, (R.OP_OR, 0, 0)], a, b), [1, 1, 1, 1, 0, NULL, 1, NULL, NULL])
    _same(_run([C0, (R.OP_NOT, 0, 0)], _col([0, 1, -5, NULL], np.int64)), [1, 0, 0, NULL])
    _same(_run([C0, (R.OP_IS_NULL, 0, 0)], _col([0, NULL], np.int64)), [0, 1])
    _same(_run([C0, (R.OP_IS_NULL, 0, 0), (R.OP_NOT, 0, 0)], _col([0.5, NULL], np.float64)), [1, 0])
    # whatever value sits under a NULL flag must not leak into AND / OR
    dirty = (np.array([7, 0], np.int64), np.array([True, True]))
    _same(_run([C0, C1, (R.OP_AND, 0, 0)], dirty, _col([0, 1], np.int64)), [0, NULL])
    _same(_run([C0, C1, (R.OP_OR, 0, 0)], dirty, _col([0, 1], np.int64)), [NULL, 1])


def test_long_arithmetic_wraps():
    a = _col([MIN, MAX, MIN, MAX, 3037000500, NULL], np.int64)
    b = _col([-1, 1, 1, MAX, 3037000500, 1], np.int64)
    _same(_run([C0, C1, (R.OP_MUL, 0, 0)], a, b), [MIN, MAX, MIN, 1, -9223372036709301616, NULL])
    _same(_run([C0, C1, (R.OP_ADD, 0, 0)], a, b), [MAX, MIN, MIN + 1, -2, 6074001000, NULL])
    _same(_run([C0, C1, (R.OP_SUB, 0, 0)], a, b), [MIN + 1, MAX - 1, MAX, 0, 0, NULL])
    _same(_run([C0, (R.OP_NEG, 0, 0)], _col([MIN, MAX, 0, 5, NULL], np.int64)), [MIN, -MAX, 0, -5, NULL])
    _same(_run([C0, (R.OP_NEG, 0, 0)], _col([0.0, -0.0, 2.5, -INF, NAN, NULL], np.float64)), [-0.0, 0.0, -2.5, INF, NAN, NULL])
    # INT columns are longs inside an expression: no 32-bit wrap
    _same(_run([C0, C0, (R.OP_MUL, 0, 0)], _col([2147483647, -2147483648], np.int32)), [4611686014132420609, 4611686018427387904])
    assert R.evaluate([C0], [_col([5], np.int32)])[0].dtype == np.int32       # alone, it passes through as INT
    assert R.evaluate([C0, C0, (R.OP_ADD, 0, 0)], [_col([5], np.int32)])[0].dtype == np.int64


def test_mixed_comparisons_widen_the_long():
    i = _col([(1 << 53) + 1, (1 << 53) + 1, MAX, MAX, MIN, 0, 0], np.int64)
    d = _col([9007199254740992.0, 9007199254740994.0, 9223372036854775808.0, INF, -9223372036854775808.0, -0.0, NAN], np.float64)
    _same(_run([C0, C1, (R.OP_EQ, 0, 0)], i, d), [1, 0, 1, 0, 1, 1, 0])        # 2^53 + 1 == 2^53 once it is a double
    _same(_run([C0, C1, (R.OP_LT, 0, 0)], i, d), [0, 1, 0, 1, 0, 0, 0])
    _same(_run([C1, C0, (R.OP_GE, 0, 0)], i, d), [1, 1, 1, 1, 1, 1, 0])
    # the same two longs compared as longs differ
    _same(_run([C0, (R.OP_CONST_I64, 0, 1 << 53), (R.OP_EQ, 0, 0)], _col([(1 << 53) + 1], np.int64)), [0])
    # long + double is a double sum of the widened long
    _same(_run([C0, C1, (R.OP_ADD, 0, 0)], _col([(1 << 53) + 1, 1], np.int64), _col([0.0, 0.5], np.float64)), [9007199254740992.0, 1.5])


def test_nan_compares_false_except_ne():
    x = _col([NAN, NAN, 1.0, NAN], np.float64)
    y = _col([NAN, 1.0, NAN, INF], np.float64)
    for op, want in ((R.OP_LT, 0), (R.OP_LE, 0), (R.OP_GT, 0), (R.OP_GE, 0), (R.OP_EQ, 0), (R.OP_NE, 1)):
        _same(_run([C0, C1, (op, 0, 0)], x, y), [want] * 4)
    z = _col([0.0, -0.0, 5e-324, -INF], np.float64)
    w = _col([-0.0, 0.0, 0.0, INF], np.float64)
    _same(_run([C0, C1, (R.OP_EQ, 0, 0)], z, w), [1, 1, 0, 0])
    _same(_run([C0, C1, (R.OP_LT, 0, 0)], z, w), [0, 0, 0, 1])
    _same(_run([C0, C1, (R.OP_GT, 0, 0)], z, w), [0, 0, 1, 0])


def test_filter_keeps_only_true_rows():
    a = _col([1, 0, NULL, 5, -1], np.int64)
    keep, out = R.apply([a], [[C0], [C0, (R.OP_CONST_I64, 0, 1), (R.OP_ADD, 0, 0)]], [C0, (R.OP_CONST_I64, 0, 0), (R.OP_GT, 0, 0)])
    assert keep.tolist() == [True, False, False, True, False]
    assert out[0][0].tolist() == [1, 5] and out[1][0].tolist() == [2, 6] and not out[0][1].any()
    keep, out = R.apply([a], [[C0, (R.OP_IS_NULL, 0, 0)]])
    assert keep.all() and out[0][0].tolist() == [0, 0, 1, 0, 0]


def test_checker_verdicts():
    I, D = (R.OP_CONST_I64, 0, 1), (R.OP_CONST_F64, 0, 1.0)
    add = (R.OP_ADD, 0, 0)
    t = [R.T_INT32, R.T_INT64, R.T_FP64]
    ok = [
        ([C0], R.T_INT32), ([C1], R.T_INT64), ([(R.OP_COL, 2, 0)], R.T_FP64), ([C0, (R.OP_NEG, 0, 0)], R.T_INT64), ([C0, C1, add], R.T_INT64),
        ([C0, D, add], R.T_FP64), ([C0, C1, (R.OP_DIV, 0, 0)], R.T_FP64), ([(R.OP_COL, 2, 0), D, (R.OP_LT, 0, 0)], R.T_INT64),
        ([(R.OP_COL, 2, 0), (R.OP_IS_NULL, 0, 0)], R.T_INT64), ([(R.OP_COL, 2, 0), (R.OP_CAST_I64, 0, 0)], R.T_INT64),
        ([C0, (R.OP_CAST_F64, 0, 0)], R.T_FP64), ([(R.OP_COL, 2, 0), (R.OP_NEG, 0, 0)], R.T_FP64),
        ([I, I, I, I, add, add, add], R.T_INT64),                                        # depth 4
        ([I] + [I, add] * 11 + [(R.OP_NEG, 0, 0)], R.T_INT64),                           # 24 instructions
    ]
    for ins, want in ok:
        assert R.check(ins, t) == (want, None), ins
    bad = [
        ([], "length"), ([I] + [I, add] * 12, "length"),                                 # 0 and 25 instructions
        ([I, I, I, I, I, add, add, add, add], "depth"),
        ([(R.OP_COL, 3, 0)], "column"), ([(R.OP_COL, -1, 0)], "column"),
        ([add], "underflow"), ([I, add], "underflow"), ([(R.OP_NOT, 0, 0)], "underflow"),
        ([D, (R.OP_NOT, 0, 0)], "logic over a double"), ([I, D, (R.OP_AND, 0, 0)], "logic over a double"),
        ([(R.OP_COL, 2, 0), I, (R.OP_OR, 0, 0)], "logic over a double"),
        ([I, I], "leaves 2 values"), ([I, (21, 0, 0)], "unknown op"), ([(0, 0, 0)], "unknown op"),
    ]
    for ins, why in bad:
        assert R.check(ins, t) == (None, why), ins
    assert R.check_scan(t, [[C0]], [(R.OP_COL, 2, 0)]) == (None, "filter: a double is not a condition")
    assert R.check_scan(t, [[C0]], [(R.OP_COL, 2, 0), D, add])[0] is None
    assert R.check_scan(t, [[C0], [add]])[0] is None and R.check_scan(t, [])[0] is None and R.check_scan(t, [[C0]] * 17)[0] is None
    assert R.check_scan(t, [[C0], [C1, D, add]], [C0, C1, (R.OP_LE, 0, 0)]) == ([R.T_INT32, R.T_FP64], None)
    assert R.check_scan(t, [[C0]] * 16)[0] == [R.T_INT32] * 16


def _wrap(v):
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >> 63 else v


def test_integer_ops_agree_with_python_int_arithmetic():
    """A second implementation: Python's unbounded ints reduced modulo 2^64, over the cross product of the edge values."""
    edge = [0, 1, -1, 2, -2, (1 << 31) - 1, -(1 << 31), 1 << 31, -(1 << 31) - 1, (1 << 53) + 1, (1 << 53) - 1, -(1 << 53) - 1, -(1 << 53) + 1,
            MIN, MAX, MIN + 1, 3037000500, -3037000500]
    pairs = list(itertools.product(edge, edge))
    a = (np.array([p[0] for p in pairs], np.int64), None)
    b = (np.array([p[1] for p in pairs], np.int64), None)
    py = {R.OP_ADD: lambda x, y: _wrap(x + y), R.OP_SUB: lambda x, y: _wrap(x - y), R.OP_MUL: lambda x, y: _wrap(x * y),
          R.OP_LT: lambda x, y: int(x < y), R.OP_LE: lambda x, y: int(x <= y), R.OP_GT: lambda x, y: int(x > y), R.OP_GE: lambda x, y: int(x >= y),
          R.OP_EQ: lambda x, y: int(x == y), R.OP_NE: lambda x, y: int(x != y)}
    for op, f in py.items():
        v, nl = R.evaluate([C0, C1, (op, 0, 0)], [a, b])
        assert not nl.any() and v.tolist() == [f(x, y) for x, y in pairs], op
    v, _ = R.evaluate([C0, (R.OP_NEG, 0, 0)], [(np.array(edge, np.int64), None)])
    assert v.tolist() == [_wrap(-x) for x in edge]
    # (double) long against Python's correctly rounded int -> float
    v, _ = R.evaluate([C0, (R.OP_CAST_F64, 0, 0)], [(np.array(edge, np.int64), None)])
    assert v.tolist() == [float(x) for x in edge]


def test_rint_cast_agrees_with_python_round():
    """Python's round() of a float is round-half-even to an exact int: a second implementation of (long) Math.rint."""
    vals = [0.5, 1.5, 2.5, 3.5, -0.5, -1.5, -2.5, 2.7, -2.7, 1e15 + 0.5, 4503599627370496.5, 4503599627370497.5, 9.3e18, -9.3e18, 9223372036854774784.0,
            -9223372036854775808.0, 1e300, -1e300, 5e-324, -5e-324, 0.0, -0.0, 123456789.5, 123456788.5]
    got = R.rint_to_long(np.array(vals, np.float64)).tolist()
    assert got == [max(MIN, min(MAX, round(v))) for v in vals]


# ------------------------------------------------------------------------------------------- the Java translator
def _java_translate():
    src = open(os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor", "operator", "gpu", "GpuExpression.java")).read()
    code = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", src, flags=re.S))
    return code[code.index("private static GpuExpression translate("):]


def test_java_translates_division_only_when_the_planner_typed_it_double():
    """integer / integer is DECIMAL in the reference (ArithmeticOperators.tdd): the GPU's DOUBLE quotient is only right for a
    call the planner typed DOUBLE / FLOAT, so every other DIVIDE must stay on the stock operator (translate returns null)."""
    code = _java_translate()
    m = re.search(r"case DIVIDE:(.*?)case LESS_THAN:", code, flags=re.S)
    assert m, "no DIVIDE case"
    body = m.group(1)
    assert "OP_DIV" in body and "return null;" in body
    assert re.search(r"call\.getType\(\)\.getSqlTypeName\(\)", body) and '"DOUBLE"' in body and '"FLOAT"' in body
    assert body.index("return null;") < body.index("op = OP_DIV;"), "the type test must come before OP_DIV is chosen"
    assert code.count("OP_DIV") == 1, "OP_DIV is emitted in one place only"
    assert "DECIMAL" in open(os.path.join(ROOT, "INTEGRATION.md")).read()


def test_java_translates_only_the_casts_the_reference_vectorises():
    """Rex2VectorizedExpressionVisitor.VECTORIZED_CAST_FUNCTION_NAMES maps BIGINT and SIGNED to CastToSigned and DOUBLE to
    CastToDouble; INTEGER and FLOAT targets are not vectorised casts there, so they are not GPU programs either."""
    code = _java_translate()
    m = re.search(r"case CAST:\s*\{(.*?)\n        \}", code, flags=re.S)
    assert m, "no CAST case"
    body = m.group(1)
    to_f64 = body[:body.index("OP_CAST_F64")]
    to_i64 = body[body.index("OP_CAST_F64"):body.index("OP_CAST_I64")]
    assert re.findall(r'"(\w+)"\.equals\(target\)', to_f64) == ["DOUBLE"]
    assert sorted(re.findall(r'"(\w+)"\.equals\(target\)', to_i64)) == ["BIGINT", "SIGNED"]
