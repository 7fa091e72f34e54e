"""The reference's vectorised expression semantics, restated in numpy for checking gsql_scan_* (Filter + Project).

A program is a postfix list of ``(op, arg, k)`` (what ``api.E.ins`` holds): it is evaluated a column at a time over
``(values, nulls)`` pairs, the way the reference evaluates one VectorizedExpression per chunk.  Nothing here imports the
product.  CG/ = polardbx-executor/src/main/codegen/, EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/.

  * INT and BIGINT operands are Java longs inside an expression: + - * wrap modulo 2^64 (done in uint64 here);
    doubles are IEEE binary64 (numpy float64);
  * a binary operator's result is NULL where either operand is (EX/vectorized/VectorizedExpressionUtils.mergeNulls);
  * + - * over a long and a double, and every comparison of one with the other, widen the long to double first (Java
    binary numeric promotion of `array1[i] op array2[i]`, CG/templates/ComparisonBinaryOperatorColumnColumn.ftl:53,
    ArithmeticBinaryOperatorColumnColumn.ftl:78); comparisons yield BIGINT 1 / 0 (LongBlock.TRUE_VALUE / FALSE_VALUE);
  * `/` is DOUBLE division and is **NULL where the divisor, as a double, equals 0** — so for 0, 0.0 and -0.0, not for NaN
    (ArithmeticBinaryOperatorColumnColumn.ftl:50-54,66-70; a zero constant divisor NULLs the whole column,
    ArithmeticBinaryOperatorColumnConst.ftl:53-55).  Integer / integer is DECIMAL in the reference
    (CG/data/ArithmeticOperators.tdd:4220 ff.) and is not a program the GPU is given;
  * unary minus is `-1 * x` (UnaryMinusOperatorColumn.ftl:48): -(+0.0) is -0.0, -INT64_MIN is INT64_MIN;
  * AND / OR are SQL's three-valued tables (LogicalBinaryOperatorColumnColumn.ftl:59-66), NOT is `x == 0` with the
    operand's NULL kept (NotOperator.ftl:48), IS NULL is never NULL (NullTestOperator.ftl);
  * CAST to BIGINT / SIGNED of a double is `(long) Math.rint(x)`: round half to even, then Java's saturating narrowing,
    NaN -> 0 (EX/vectorized/build/Rex2VectorizedExpressionVisitor.java:127-135 binds both to CastToSigned,
    CG/templates/CastNumericSigned.ftl:61,70); of a long it is the identity.  CAST to DOUBLE of a long is Java's
    `(double) x`, round to nearest even;
  * a filter keeps the rows where the condition is TRUE: not FALSE, not NULL (EX/operator/VectorizedFilterExec.java).

Java has one NaN as far as these operators can tell (Double.doubleToLongBits canonicalises it), so same_columns compares
doubles bit for bit with every NaN mapped to one pattern; +0.0 and -0.0 stay different.

check() restates what include/gsql_gpu.h promises gsql_scan_create accepts: 1..24 instructions, an operand stack of at
most 4, NOT / AND / OR over integers only, a filter that is not a DOUBLE.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

T_INT32, T_INT64, T_FP64 = 0, 1, 2
(OP_COL, OP_CONST_I64, OP_CONST_F64, OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_NEG, OP_LT, OP_LE, OP_GT, OP_GE, OP_EQ, OP_NE, OP_AND, OP_OR,
 OP_NOT, OP_IS_NULL, OP_CAST_F64, OP_CAST_I64) = range(1, 21)
MAX_INS, MAX_STACK, MAX_OUT = 24, 4, 16
ARITH = (OP_ADD, OP_SUB, OP_MUL, OP_DIV)
COMPARE = (OP_LT, OP_LE, OP_GT, OP_GE, OP_EQ, OP_NE)
LOGIC = (OP_AND, OP_OR)
UNARY = (OP_NEG, OP_NOT, OP_IS_NULL, OP_CAST_F64, OP_CAST_I64)
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
_NP = {T_INT32: np.int32, T_INT64: np.int64, T_FP64: np.float64}

Col = Tuple[np.ndarray, Optional[np.ndarray]]
Ins = Tuple[int, int, object]


# --------------------------------------------------------------------------------------------------- type checker
def check(ins: Sequence[Ins], in_types: Sequence[int]) -> Tuple[Optional[int], Optional[str]]:
    """-> (result type, None), or (None, why the program is refused)."""
    if not 1 <= len(ins) <= MAX_INS:
        return None, "length"
    st: List[bool] = []  # is the slot a double
    for op, arg, _ in ins:
        if op in (OP_COL, OP_CONST_I64, OP_CONST_F64):
            if op == OP_COL and not 0 <= arg < len(in_types):
                return None, "column"
            if len(st) >= MAX_STACK:
                return None, "depth"
            st.append(in_types[arg] == T_FP64 if op == OP_COL else op == OP_CONST_F64)
        elif op in UNARY:
            if len(st) < 1:
                return None, "underflow"
            if op == OP_NOT and st[-1]:
                return None, "logic over a double"
            st[-1] = st[-1] if op == OP_NEG else op == OP_CAST_F64
        elif op in ARITH or op in COMPARE or op in LOGIC:
            if len(st) < 2:
                return None, "underflow"
            b, a = st.pop(), st.pop()
            if op in LOGIC and (a or b):
                return None, "logic over a double"
            st.append(op in ARITH and (a or b or op == OP_DIV))
        else:
            return None, "unknown op"
    if len(st) != 1:
        return None, "leaves %d values" % len(st)
    if len(ins) == 1 and ins[0][0] == OP_COL:
        return in_types[ins[0][1]], None  # a lone column passes through with its own type
    return (T_FP64 if st[0] else T_INT64), None


def check_scan(in_types: Sequence[int], outs: Sequence[Sequence[Ins]], filt: Optional[Sequence[Ins]] = None):
    """-> (output types, None), or (None, reason): the verdict on a whole gsql_scan_spec."""
    if not 1 <= len(outs) <= MAX_OUT:
        return None, "outputs"
    if filt is not None:
        t, why = check(filt, in_types)
        if t is None:
            return None, "filter: " + why
        if t == T_FP64:
            return None, "filter: a double is not a condition"
    types = []
    for e in outs:
        t, why = check(e, in_types)
        if t is None:
            return None, why
        types.append(t)
    return types, None


# ------------------------------------------------------------------------------------------------------ evaluator
def _u(x: np.ndarray) -> np.ndarray:
    return x.view(np.uint64)


def long_to_double(x: np.ndarray) -> np.ndarray:
    """Java (double) long: round to nearest, ties to even."""
    return x.astype(np.float64)


def rint_to_long(d: np.ndarray) -> np.ndarray:
    """(long) Math.rint(d): half to even, saturating at the ends of long, NaN -> 0."""
    r = np.rint(d)
    hi, lo, nan = r >= 9223372036854775808.0, r <= -9223372036854775808.0, np.isnan(r)
    v = np.where(hi | lo | nan, 0.0, r).astype(np.int64)
    v[hi] = INT64_MAX
    v[lo] = INT64_MIN
    return v


def _as_f(v: np.ndarray, isf: bool) -> np.ndarray:
    return v if isf else long_to_double(v)


def evaluate(ins: Sequence[Ins], cols: Sequence[Col], n: Optional[int] = None):
    """-> (values, nulls): int64 or float64 values for every row (INT32 for a lone INT column); the values under a NULL
    flag mean nothing."""
    n = len(cols[0][0]) if n is None else n
    in_types = [{np.dtype(np.int32): T_INT32, np.dtype(np.int64): T_INT64, np.dtype(np.float64): T_FP64}[np.asarray(d).dtype] for d, _ in cols]
    t, why = check(ins, in_types)
    assert t is not None, why
    st: List[Tuple[np.ndarray, np.ndarray, bool]] = []
    with np.errstate(all="ignore"):
        for op, arg, k in ins:
            if op == OP_COL:
                d, nl = cols[arg]
                d = np.asarray(d)
                isf = d.dtype == np.float64
                st.append((d if isf else d.astype(np.int64), np.zeros(n, bool) if nl is None else np.asarray(nl).astype(bool), isf))
            elif op == OP_CONST_I64:
                st.append((np.full(n, int(k), np.int64), np.zeros(n, bool), False))
            elif op == OP_CONST_F64:
                st.append((np.full(n, float(k), np.float64), np.zeros(n, bool), True))
            elif op == OP_NEG:
                v, nl, isf = st.pop()
                st.append((-1.0 * v if isf else (_u(np.full(n, -1, np.int64)) * _u(v)).view(np.int64), nl, isf))
            elif op == OP_NOT:
                v, nl, _ = st.pop()
                st.append(((v == 0).astype(np.int64), nl, False))
            elif op == OP_IS_NULL:
                v, nl, _ = st.pop()
                st.append((nl.astype(np.int64), np.zeros(n, bool), False))
            elif op == OP_CAST_F64:
                v, nl, isf = st.pop()
                st.append((_as_f(v, isf), nl, True))
            elif op == OP_CAST_I64:
                v, nl, isf = st.pop()
                st.append((rint_to_long(v) if isf else v, nl, False))
            elif op in LOGIC:
                b, bn, _ = st.pop()
                a, an, _ = st.pop()
                b1, b2 = a != 0, b != 0
                if op == OP_AND:
                    nl = (an & bn) | (an & b2) | (bn & b1)
                    v = ~((~an & ~b1) | (~bn & ~b2))
                else:
                    nl = (an & bn) | (an & ~b2) | (bn & ~b1)
                    v = (~an & b1) | (~bn & b2)
                st.append((v.astype(np.int64), nl, False))
            else:
                b, bn, bf = st.pop()
                a, an, af = st.pop()
                nl = an | bn
                if af or bf or op == OP_DIV:
                    x, y = _as_f(a, af), _as_f(b, bf)
                    if op == OP_DIV:
                        nl = nl | (y == 0)
                    v = {OP_ADD: lambda: x + y, OP_SUB: lambda: x - y, OP_MUL: lambda: x * y, OP_DIV: lambda: x / y, OP_LT: lambda: x < y,
                         OP_LE: lambda: x <= y, OP_GT: lambda: x > y, OP_GE: lambda: x >= y, OP_EQ: lambda: x == y, OP_NE: lambda: x != y}[op]()
                else:
                    v = {OP_ADD: lambda: (_u(a) + _u(b)).view(np.int64), OP_SUB: lambda: (_u(a) - _u(b)).view(np.int64),
                         OP_MUL: lambda: (_u(a) * _u(b)).view(np.int64), OP_LT: lambda: a < b, OP_LE: lambda: a <= b, OP_GT: lambda: a > b,
                         OP_GE: lambda: a >= b, OP_EQ: lambda: a == b, OP_NE: lambda: a != b}[op]()
                st.append((v.astype(np.int64) if op in COMPARE else v, nl, op in ARITH and (af or bf or op == OP_DIV)))
    v, nl, _ = st.pop()
    return v.astype(_NP[t]), nl


def apply(cols: Sequence[Col], outs: Sequence[Sequence[Ins]], filt: Optional[Sequence[Ins]] = None):
    """-> (kept-row mask, output columns over the kept rows, in input order)."""
    n = len(cols[0][0])
    keep = np.ones(n, bool)
    if filt is not None:
        v, nl = evaluate(filt, cols, n)
        keep = ~nl & (v != 0)
    res = []
    for e in outs:
        v, nl = evaluate(e, cols, n)
        res.append((v[keep], nl[keep]))
    return keep, res


# ----------------------------------------------------------------------------------------------------- comparison
def canon_bits(d: np.ndarray) -> np.ndarray:
    """Double.doubleToLongBits: the bit pattern, every NaN as 0x7ff8000000000000."""
    d = np.ascontiguousarray(d, dtype=np.float64)
    b = d.view(np.uint64).copy()
    b[np.isnan(d)] = np.uint64(0x7ff8000000000000)
    return b


def same_columns(got: Sequence[Col], exp: Sequence[Col], what: str = "") -> None:
    """Row by row: NULL flags exactly, types exactly, values bit for bit wherever the row is not NULL."""
    assert len(got) == len(exp), (what, len(got), len(exp))
    for c, ((gd, gn), (ed, en)) in enumerate(zip(got, exp)):
        gd, ed = np.asarray(gd), np.asarray(ed)
        assert gd.dtype == ed.dtype, f"{what} column {c}: type {gd.dtype}, expected {ed.dtype}"
        assert len(gd) == len(ed), f"{what} column {c}: {len(gd)} rows, expected {len(ed)}"
        gn = np.zeros(len(gd), bool) if gn is None else np.asarray(gn).astype(bool)
        en = np.zeros(len(ed), bool) if en is None else np.asarray(en).astype(bool)
        bad = np.flatnonzero(gn != en)
        assert bad.size == 0, f"{what} column {c}: NULL flag differs at rows {bad[:8].tolist()} (got {gn[bad[:8]].tolist()})"
        g, e = (canon_bits(gd), canon_bits(ed)) if gd.dtype == np.float64 else (gd, ed)
        bad = np.flatnonzero((g != e) & ~en)
        assert bad.size == 0, f"{what} column {c}: rows {bad[:8].tolist()} got {gd[bad[:8]].tolist()} expected {ed[bad[:8]].tolist()}"
