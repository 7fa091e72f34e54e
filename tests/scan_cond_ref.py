"""CASE, COALESCE, IN, BETWEEN and DATE comparisons as the reference evaluates them, restated in numpy for checking
gsql_scan_create2 (ops 32..36 of include/gsql_gpu.h).  Nothing here imports the product.

EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/, CG/ = polardbx-executor/src/main/codegen/.

Two layers:

* ``ref_*``: each reference class as it reads, over ``(values, nulls)`` columns and Python constants (None = a NULL
  literal).  These are what the hand-worked tests pin;
* ``evaluate`` / ``check`` / ``check_scan``: the postfix programs the GPU runs (scan_ref's ops plus the five new ones),
  which the translator builds from those classes.  ``evaluate`` takes old ops from tests/scan_ref.py unchanged.

The rules, and the quirks kept:

* CASE (EX/vectorized/CaseVectorizedExpression.java:74-120): children are ``when, then, ..., else``; each when narrows
  the rows still open by conditionalEval (VectorizedExpressionUtils.java:217-240), so the first TRUE condition wins and
  a NULL or FALSE one is not taken.  Rex2VectorizedExpressionVisitor.java:458-470 wraps every condition that cannot bind
  a filter-mode comparison in IS TRUE, so every condition selects exactly its TRUE rows.  Calcite gives a CASE without
  ELSE a NULL literal as its last operand.
* COALESCE (EX/vectorized/CoalesceVectorizedExpression.java:62-107): the first non-NULL argument, NULL if none is.
* IN (EX/vectorized/compare/AbstractInLongColLongConstVectorizedExpression.java): a NULL constant makes every row NULL
  (lines 90-97); otherwise ``anyMatch(value)`` (67-74, 99-111) with no NULL merge, so a NULL row compares the value
  stored under its flag: 0 from every stock BlockBuilder.appendNull, and 0 from k_scan's column load — ``NULL IN (0, 5)``
  is TRUE.  Classes exist for 1..100 constants (CG/data/InColConstOperators.tdd: operandCount counts the constants;
  CG/templates/InColumnConst.ftl:21-42 adds the column).
* BETWEEN (EX/vectorized/compare/BetweenLongColLongConstLongConstVectorizedExpression.java): the same NULL rules
  (78-85), ``x >= lo && x <= hi`` (93-96, 101-104).
* DATE column <cmp> CHAR constant (CG/templates/ComparisonBinaryDateColumnConst.ftl:40-48, 64-93 with
  CG/data/DateComparisonOperators.tdd: GT GE LT LE EQ NE, constType Char only): the constant is
  ``TimeStorage.writeDate(DateType.convertFrom(literal))`` and the rows compare packed longs, NULL merged from the
  column; a NULL constant makes every row NULL.  A DATE-typed literal matches no vectorised class (its argument type is
  Date, Rex2ArgumentInfo.java:68-71), and DATE col vs DATE col (GT / LT only) reads the right operand at the
  selection's ordinal, not its position (LTDateColDateColVectorizedExpression.java:63-66): neither is translated.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from tests import scan_ref as R

OP_CONST_NULL, OP_CASE_WHEN, OP_COALESCE, OP_BETWEEN, OP_IN = range(32, 37)
NEW_OPS = (OP_CONST_NULL, OP_CASE_WHEN, OP_COALESCE, OP_BETWEEN, OP_IN)
MAX_IN_LIST, MAX_SCAN_POOL = 256, 1024
REF_MAX_IN_CONSTANTS = 100  # the last operandCount of InColConstOperators.tdd

Col = Tuple[np.ndarray, np.ndarray]


def _nl(c, n):
    return np.zeros(n, bool) if c[1] is None else np.asarray(c[1]).astype(bool)


# --------------------------------------------------------------------------------------- the reference classes
def ref_case(whens: Sequence[Col], thens: Sequence[Col], else_: Optional[Col]) -> Col:
    """CaseVectorizedExpression over evaluated children; else_ None is the NULL literal Calcite supplies."""
    n = len(whens[0][0])
    dt = np.asarray(thens[0][0]).dtype
    out, nulls = np.zeros(n, dt), np.ones(n, bool)
    open_ = np.ones(n, bool)
    for w, t in zip(whens, thens):
        take = open_ & ~_nl(w, n) & (np.asarray(w[0]) != 0)
        out[take], nulls[take] = np.asarray(t[0])[take], _nl(t, n)[take]
        open_ &= ~take
    if else_ is not None:
        out[open_], nulls[open_] = np.asarray(else_[0])[open_], _nl(else_, n)[open_]
    return out, nulls


def ref_coalesce(args: Sequence[Col]) -> Col:
    n = len(args[0][0])
    out, nulls = np.zeros(n, np.asarray(args[0][0]).dtype), np.ones(n, bool)
    for a in args:
        take = nulls & ~_nl(a, n)
        out[take] = np.asarray(a[0])[take]
        nulls &= ~take
    return out, nulls


def ref_in(col: Col, consts: Sequence[Optional[int]]) -> Col:
    """col: a column block (values under a NULL flag as the block holds them)."""
    n = len(col[0])
    if any(c is None for c in consts):
        return np.zeros(n, np.int64), np.ones(n, bool)
    v = np.asarray(col[0]).astype(np.int64)
    return np.isin(v, np.array(consts, np.int64)).astype(np.int64), np.zeros(n, bool)


def ref_between(col: Col, lo: Optional[int], hi: Optional[int]) -> Col:
    n = len(col[0])
    if lo is None or hi is None:
        return np.zeros(n, np.int64), np.ones(n, bool)
    v = np.asarray(col[0]).astype(np.int64)
    return ((v >= lo) & (v <= hi)).astype(np.int64), np.zeros(n, bool)


def write_date(y: int, m: int, d: int) -> int:
    """TimeStorage.writeDate (polardbx-common .../time/core/TimeStorage.java:170-173)."""
    return (((y * 13 + m) << 5) | d) << 41


def pack_days(days: np.ndarray) -> np.ndarray:
    """Days since 1970-01-01 -> the DateBlock packed long of that date."""
    dt = np.asarray(days).astype("datetime64[D]")
    y = dt.astype("datetime64[Y]").astype(np.int64) + 1970
    m = dt.astype("datetime64[M]").astype(np.int64) % 12 + 1
    d = (dt - dt.astype("datetime64[M]")).astype(np.int64) + 1
    return (((y * 13 + m) << 5) | d) << 41


_CMP = {R.OP_LT: np.less, R.OP_LE: np.less_equal, R.OP_GT: np.greater, R.OP_GE: np.greater_equal, R.OP_EQ: np.equal, R.OP_NE: np.not_equal}


def ref_date_cmp(col: Col, op: int, packed: Optional[int]) -> Col:
    """ComparisonBinaryDateColumnConst over a DateBlock; packed: the converted constant, None for a NULL literal."""
    n = len(col[0])
    if packed is None:
        return np.zeros(n, np.int64), np.ones(n, bool)
    return _CMP[op](np.asarray(col[0], np.int64), packed).astype(np.int64), _nl(col, n)


# ------------------------------------------------------------------------------------------- the GPU programs
def _consts(arg, k, pool):
    """IN / BETWEEN constants: api.E keeps them in the instruction as a tuple; a raw spec points into the pool."""
    return list(k) if isinstance(k, tuple) else list(pool[arg:arg + k])


def check(ins, in_types, npool: int = 0, used: Optional[List[int]] = None):
    """gsql_scan_create2's verdict on one program -> (result type, None) or (None, why).  used[0] accumulates the pool
    entries the program's IN lists and BETWEENs take."""
    if not 1 <= len(ins) <= R.MAX_INS:
        return None, "length"
    used = [0] if used is None else used
    st: List[bool] = []
    for op, arg, k in ins:
        if op in (R.OP_COL, R.OP_CONST_I64, R.OP_CONST_F64, OP_CONST_NULL):
            if op == R.OP_COL and not 0 <= arg < len(in_types):
                return None, "column"
            if op == OP_CONST_NULL and arg not in (R.T_INT64, R.T_FP64):
                return None, "null type"
            if len(st) >= R.MAX_STACK:
                return None, "depth"
            st.append({R.OP_COL: lambda: in_types[arg] == R.T_FP64, R.OP_CONST_I64: lambda: False, R.OP_CONST_F64: lambda: True,
                       OP_CONST_NULL: lambda: arg == R.T_FP64}[op]())
        elif op in R.UNARY:
            if len(st) < 1:
                return None, "underflow"
            if op == R.OP_NOT and st[-1]:
                return None, "logic over a double"
            st[-1] = st[-1] if op == R.OP_NEG else op == R.OP_CAST_F64
        elif op in R.ARITH or op in R.COMPARE or op in R.LOGIC:
            if len(st) < 2:
                return None, "underflow"
            b, a = st.pop(), st.pop()
            if op in R.LOGIC and (a or b):
                return None, "logic over a double"
            st.append(op in R.ARITH and (a or b or op == R.OP_DIV))
        elif op == OP_CASE_WHEN:
            if len(st) < 3:
                return None, "underflow"
            if st[-2]:
                return None, "condition is a double"
            if st[-3] != st[-1]:
                return None, "branch types"
            st.pop(), st.pop()
        elif op == OP_COALESCE:
            if len(st) < 2:
                return None, "underflow"
            if st[-2] != st[-1]:
                return None, "branch types"
            st.pop()
        elif op in (OP_BETWEEN, OP_IN):
            if len(st) < 1:
                return None, "underflow"
            if st[-1]:
                return None, "set over a double"
            cnt = 2 if op == OP_BETWEEN else (len(k) if isinstance(k, tuple) else k)
            if not 1 <= cnt <= MAX_IN_LIST:
                return None, "list length"
            if not isinstance(k, tuple) and (arg < 0 or arg + cnt > npool):
                return None, "pool range"
            if used[0] + cnt > MAX_SCAN_POOL:
                return None, "pool size"
            used[0] += cnt
        else:
            return None, "unknown op"
    if len(st) != 1:
        return None, "leaves %d values" % len(st)
    if len(ins) == 1 and ins[0][0] == R.OP_COL:
        return in_types[ins[0][1]], None
    return (R.T_FP64 if st[0] else R.T_INT64), None


def check_scan(in_types, outs, filt=None, npool: int = 0):
    """-> (output types, None) or (None, reason): gsql_scan_create2 on a whole spec (filter first, then the outputs)."""
    if not 1 <= len(outs) <= R.MAX_OUT:
        return None, "outputs"
    if not 0 <= npool <= MAX_SCAN_POOL:
        return None, "pool"
    used = [0]
    if filt is not None:
        t, why = check(filt, in_types, npool, used)
        if t is None:
            return None, "filter: " + why
        if t == R.T_FP64:
            return None, "filter: a double is not a condition"
    types = []
    for e in outs:
        t, why = check(e, in_types, npool, used)
        if t is None:
            return None, why
        types.append(t)
    return types, None


def evaluate(ins, cols, pool: Sequence[int] = (), n: Optional[int] = None):
    """-> (values, nulls) of a program: old ops evaluated by scan_ref one at a time over the stack's columns; values under
    a NULL flag mean nothing, except that IN and BETWEEN read such a row as 0."""
    n = len(cols[0][0]) if n is None else n
    in_types = [{np.dtype(np.int32): R.T_INT32, np.dtype(np.int64): R.T_INT64, np.dtype(np.float64): R.T_FP64}[np.asarray(d).dtype] for d, _ in cols]
    t, why = check(ins, in_types, len(pool))
    assert t is not None, why
    if len(ins) == 1 and ins[0][0] == R.OP_COL:
        return R.evaluate(ins, cols, n)
    st: List[Col] = []
    for op, arg, k in ins:
        if op == R.OP_COL:
            d, nl = cols[arg]
            d = np.asarray(d)
            st.append((d if d.dtype == np.float64 else d.astype(np.int64), _nl((d, nl), n)))
        elif op in (R.OP_CONST_I64, R.OP_CONST_F64):
            st.append(R.evaluate([(op, 0, k)], cols, n))
        elif op in R.UNARY:
            st.append(R.evaluate([(R.OP_COL, 0, 0), (op, 0, 0)], [st.pop()], n))
        elif op in R.ARITH or op in R.COMPARE or op in R.LOGIC:
            b = st.pop()
            a = st.pop()
            st.append(R.evaluate([(R.OP_COL, 0, 0), (R.OP_COL, 1, 0), (op, 0, 0)], [a, b], n))
        elif op == OP_CONST_NULL:
            st.append((np.zeros(n, np.float64 if arg == R.T_FP64 else np.int64), np.ones(n, bool)))
        elif op == OP_CASE_WHEN:
            then, cond, acc = st.pop(), st.pop(), st.pop()
            st.append(ref_case([cond], [then], acc))
        elif op == OP_COALESCE:
            b, a = st.pop(), st.pop()
            st.append(ref_coalesce([a, b]))
        else:
            v, nl = st.pop()
            x = (np.where(nl, 0, v), None)
            c = _consts(arg, k, pool)
            st.append(ref_between(x, c[0], c[1]) if op == OP_BETWEEN else ref_in(x, c))
    v, nl = st.pop()
    return v.astype(R._NP[t]), nl


def apply(cols, outs, filt=None, pool: Sequence[int] = ()):
    """-> (kept-row mask, output columns over the kept rows, in input order)."""
    n = len(cols[0][0])
    keep = np.ones(n, bool)
    if filt is not None:
        v, nl = evaluate(filt, cols, pool, n)
        keep = ~nl & (v != 0)
    res = []
    for e in outs:
        v, nl = evaluate(e, cols, pool, n)
        res.append((v[keep], nl[keep]))
    return keep, res
