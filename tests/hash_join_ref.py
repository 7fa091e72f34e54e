"""ParallelHashJoinExec by definition: a row-level restatement of what a hash join returns, with no hash table.

This is the yardstick the join tests hold both the GPU (gsql_join_*) and the CPU oracle (oracle.c) against.  It
shares no code with either: the oracle restates the reference's Java hash table, this file states the result.

Columns are ``(values, nulls)`` pairs (numpy arrays, ``nulls`` None or bool/uint8, non-zero = NULL).  ``spec`` is an
``oracle.JoinSpec`` (only its fields are read).  The rules:

* Keys.  Each key component is converted to its unified type (EX/chunk/Converters.java): integer widening, or the
  ``(double)`` cast, so a BIGINT above 2^53 rounds to the nearest double.  A NULL component never matches.  A DOUBLE
  component matches by bit identity: -0.0 matches only -0.0, +0.0 only +0.0, and NaN (any payload) matches nothing.
  (The reference's own answer for ±0.0 depends on its bucket count -- see test_hash_join_ref_cpu.py -- and is
  the bit-identity answer for every build side above 8192 rows.)
* Output schema (AbstractJoinExec.java:103-120): SEMI / ANTI -> outer; single join -> outer || first inner column;
  RIGHT -> inner || outer; INNER / LEFT -> outer || inner.
* Condition: ``cond_ne`` = AND_i (col_i IS NULL OR col_i != v_i) over the join row leftSide || rightSide (inner ||
  outer for RIGHT, else outer || inner), evaluated per key-matched pair before the pair counts as a match.
* Single join (max_one_row): a second passing match of one outer row raises MoreThanOneRow.
* LEFT / RIGHT: an outer row with no passing match is emitted once, NULL-padded on the inner side.
* SEMI: an outer row with a passing match.  ANTI: an outer row without one; with anti operands (NOT IN) a row whose
  operand is NULL is dropped, and when the build side is exactly one column holding a NULL the result is empty
  (AbstractBufferedJoinExec.doSpecialCheckForSemiJoin:290-309).
* Empty build side: INNER and SEMI return nothing; ANTI passes every outer row, NULL operands included.
* build_outer only changes which side is hashed: the outer side is the build side and its unmatched rows are emitted
  NULL-padded after the probe, so the rows are those of the same join without it.
"""
from __future__ import annotations

from collections import Counter
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

Col = Tuple[np.ndarray, Optional[np.ndarray]]

T_INT32, T_INT64, T_FP64 = 0, 1, 2
INNER, LEFT, RIGHT, SEMI, ANTI = 0, 1, 2, 3, 4


class MoreThanOneRow(RuntimeError):
    """ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW."""


class Unsupported(ValueError):
    """A combination the hash join does not take (gsql_join_create refuses it)."""


def _nulls(col: Col) -> np.ndarray:
    data, nulls = col
    n = len(data)
    return np.zeros(n, bool) if nulls is None else np.asarray(nulls).astype(bool)


def key_tuples(cols: Sequence[Col], key_cols: Sequence[int], key_types: Sequence[int]) -> List[Optional[tuple]]:
    """Per row: the tuple of key components in the unified types (a DOUBLE as its 64-bit pattern), or None when the
    row can never match (a NULL or NaN component)."""
    n = len(cols[0][0])
    valid = np.ones(n, bool)
    parts = []
    for c, t in zip(key_cols, key_types):
        data = np.asarray(cols[c][0])
        valid &= ~_nulls(cols[c])
        if t == T_FP64:
            d = data.astype(np.float64)  # Converters: (double) cast, round to nearest
            valid &= ~np.isnan(d)
            parts.append(d.view(np.int64))
        else:
            if data.dtype.kind != "i" or (t == T_INT32 and data.dtype != np.int32):
                raise Unsupported("narrowing key conversion")
            parts.append(data.astype(np.int64))
    tuples = list(zip(*[p.tolist() for p in parts]))
    return [k if v else None for k, v in zip(tuples, valid.tolist())]


def output_schema(spec, n_outer: int, n_inner: int) -> List[Tuple[str, int]]:
    """[(side, column)] of the output, side 'o' (outer) or 'i' (inner)."""
    outer = [("o", c) for c in range(n_outer)]
    inner = [("i", c) for c in range(n_inner)]
    if spec.join_type in (SEMI, ANTI):
        return outer
    if spec.max_one_row:
        return outer + inner[:1]
    if spec.join_type == RIGHT:
        return inner + outer
    return outer + inner


def _check_spec(spec, outer: Sequence[Col], inner: Sequence[Col]):
    semi = spec.join_type in (SEMI, ANTI)
    if semi and spec.max_one_row:
        raise Unsupported("single (max-one-row) semi/anti join")
    if spec.build_outer and (semi or spec.cond_ne):
        raise Unsupported("build_outer with semi/anti/condition")
    if spec.build_outer and spec.max_one_row:
        raise Unsupported("build_outer single join")
    left, right = (inner, outer) if spec.join_type == RIGHT else (outer, inner)
    for c, _ in spec.cond_ne:
        col = left[c] if c < len(left) else right[c - len(left)]
        if np.asarray(col[0]).dtype == np.float64:
            raise Unsupported("condition on a double column")


def hash_join(spec, outer: Sequence[Col], inner: Sequence[Col]) -> List[Col]:
    """The join's output rows (order unspecified) as columns of the output schema, NULLs with value 0."""
    _check_spec(spec, outer, inner)
    jt = spec.join_type
    n_outer, n_inner = len(outer[0][0]), len(inner[0][0])
    schema = output_schema(spec, len(outer), len(inner))
    pairs_o: List[int] = []
    pairs_i: List[int] = []  # -1: NULL-padded inner side

    def done():
        return _gather(schema, outer, inner, pairs_o, pairs_i)

    if n_inner == 0:
        if jt == ANTI:
            pairs_o.extend(range(n_outer))
            pairs_i.extend([-1] * n_outer)
            return done()
        if jt in (INNER, SEMI):
            return done()
    if jt == ANTI and spec.anti_operands and len(inner) == 1 and _nulls(inner[0]).any():
        return done()  # x NOT IN (..., NULL, ...) is never true

    okeys = key_tuples(outer, spec.outer_keys, spec.key_types)
    ikeys = key_tuples(inner, spec.inner_keys, spec.key_types)
    index: Dict[tuple, List[int]] = {}
    for m, k in enumerate(ikeys):
        if k is not None:
            index.setdefault(k, []).append(m)

    # condition columns of the join row, resolved to (side, column)
    nleft = len(inner) if jt == RIGHT else len(outer)
    lside, rside = ("i", "o") if jt == RIGHT else ("o", "i")
    conds = []
    for c, v in spec.cond_ne:
        side, col = (lside, c) if c < nleft else (rside, c - nleft)
        src = outer if side == "o" else inner
        conds.append((side, np.asarray(src[col][0]).astype(np.int64).tolist(), _nulls(src[col]).tolist(), int(v)))

    def passes(r: int, m: int) -> bool:
        for side, vals, nl, v in conds:
            row = r if side == "o" else m
            if not nl[row] and vals[row] == v:
                return False
        return True

    anti_nulls = [_nulls(outer[c]) for c in (spec.anti_operands or [])]
    anti_drop = np.zeros(n_outer, bool)
    for a in anti_nulls:
        anti_drop |= a
    anti_drop = anti_drop.tolist()

    for r, k in enumerate(okeys):
        cands = index.get(k, ()) if k is not None else ()
        hits = [m for m in cands if passes(r, m)] if conds else list(cands)
        if spec.max_one_row and len(hits) > 1:
            raise MoreThanOneRow()
        if jt in (INNER, LEFT, RIGHT):
            pairs_o.extend([r] * len(hits))
            pairs_i.extend(hits)
            if not hits and jt != INNER:
                pairs_o.append(r)
                pairs_i.append(-1)
        elif jt == SEMI:
            if hits:
                pairs_o.append(r)
                pairs_i.append(-1)
        elif not hits and not anti_drop[r]:
            pairs_o.append(r)
            pairs_i.append(-1)
    return done()


def _gather(schema, outer, inner, pairs_o, pairs_i) -> List[Col]:
    po = np.asarray(pairs_o, dtype=np.int64)
    pi = np.asarray(pairs_i, dtype=np.int64)
    out = []
    for side, c in schema:
        src, idx = (outer, po) if side == "o" else (inner, pi)
        data = np.asarray(src[c][0])
        pad = idx < 0
        safe = np.where(pad, 0, idx)
        if len(data):
            vals, nl = data[safe], pad | _nulls(src[c])[safe]
        else:
            vals, nl = np.zeros(len(idx), data.dtype), np.ones(len(idx), bool)
        vals[nl] = 0  # a gather copies bits: NaN payloads and signed zeros survive
        out.append((vals, nl))
    return out


# ---------------------------------------------------------------------------------------------- bit-exact rows
def _col_bits(col: Col) -> list:
    data, _ = col
    data = np.asarray(data)
    vals = (data.view(np.int64) if data.dtype == np.float64 else data.astype(np.int64)).tolist()
    nl = _nulls(col).tolist()
    return [None if isnull else v for v, isnull in zip(vals, nl)]


def rows_bits(cols: Sequence[Col]) -> Counter:
    """Order-insensitive row multiset in which a DOUBLE counts by its 64-bit pattern (so -0.0 != +0.0 and NaN
    payloads count) and a NULL's value bits are ignored."""
    if not cols:
        return Counter()
    return Counter(zip(*[_col_bits(c) for c in cols]))


def assert_rows_equal(got: Sequence[Col], exp: Sequence[Col], what: str = ""):
    """Same column count and types, and the same rows bit for bit (as multisets)."""
    assert len(got) == len(exp), f"{what}: {len(got)} columns, expected {len(exp)}"
    for c, (g, e) in enumerate(zip(got, exp)):
        assert np.asarray(g[0]).dtype == np.asarray(e[0]).dtype, f"{what}: column {c} type {np.asarray(g[0]).dtype}"
    ng = len(got[0][0]) if got else 0
    ne = len(exp[0][0]) if exp else 0
    a, b = rows_bits(got), rows_bits(exp)
    if a != b:
        extra, missing = list((a - b).items())[:5], list((b - a).items())[:5]
        raise AssertionError(f"{what}: {ng} rows, expected {ne}; unexpected {extra}; missing {missing}")
