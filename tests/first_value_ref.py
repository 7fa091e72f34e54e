"""Restatement of __FIRST_VALUE (EX/calc/aggfunctions/InternalFirstValue.java) in the reference's two aggregations, for
checking GSQL_AGG_FIRST_VALUE:

  hash (AggOpenHashMap.putChunk:100-139 + InternalFirstValue.accumulate:96-108 / writeResultTo:112-127)
    * rows are accumulated in consume order, position order within a batch; a group's value is that of the first row
      accumulated into it, NULL included (the value buffer appends when groupId == size());
    * one-group rule: when the aggregation ends with exactly one group (always so without keys), the value is the first
      non-NULL one accumulated into group 0 (fixScalarAggValue), NULL if none;
    * no keys and no rows: one row, NULL.
  sorted (SortAggExec.java:90-122: every group is group 0, reset in between)
    * every group's value is its first non-NULL one, NULL if all are NULL.

A value is None (NULL) or its bits as a Python int: INT / BIGINT by value, DOUBLE as the int64 image of its bits.
`hash_literal` / `sorted_literal` walk rows one at a time; `hash_np` / `sorted_np` state the same rules over numpy arrays
for large inputs.
"""
from __future__ import annotations

import itertools
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from tests import agg_exact as ax
from tests import sortagg_ref as sref


def _nulls(c) -> np.ndarray:
    d, nl = c
    return np.zeros(len(d), bool) if nl is None else np.asarray(nl, bool)


def value_bits(d: np.ndarray) -> np.ndarray:
    d = np.asarray(d)
    return d.view(np.int64) if d.dtype == np.float64 else d.astype(np.int64)


def _value(c, r) -> Optional[int]:
    return None if _nulls(c)[r] else int(value_bits(c[0])[r])


def _hash_key(cols, groups, r) -> tuple:
    """The hash aggregation's key: NULL, the integer, or a DOUBLE's canonical image (-0.0 = +0.0, one NaN)."""
    out = []
    for g in groups:
        nl = _nulls(cols[g])
        out.append(None if nl[r] else int(ax._key_image(np.asarray(cols[g][0])[r:r + 1], nl[r:r + 1])[0]))
    return tuple(out)


def hash_literal(batches: Sequence[Sequence[Tuple]], groups: Sequence[int], vcols: Sequence[int]) -> Dict[tuple, List]:
    """-> {group key: [value per FIRST_VALUE column]}."""
    gid_of: Dict[tuple, int] = {} if groups else {(): 0}
    first: List[List] = [[] for _ in vcols]
    fix: List[Optional[int]] = [None] * len(vcols)
    for cols in batches:
        for pos in range(len(cols[0][0]) if cols else 0):
            gid = gid_of.setdefault(_hash_key(cols, groups, pos), len(gid_of)) if groups else 0
            for i, v in enumerate(vcols):
                val = _value(cols[v], pos)
                if gid == 0 and fix[i] is None and val is not None:
                    fix[i] = val
                if gid == len(first[i]):
                    first[i].append(val)
    out = {}
    for k, gid in gid_of.items():
        out[k] = [None if not first[i] else (fix[i] if len(first[i]) == 1 else first[i][gid]) for i in range(len(vcols))]
    return out


def _concat(batches):
    if not batches:
        return []
    return [(np.concatenate([np.asarray(b[c][0]) for b in batches]), np.concatenate([_nulls(b[c]) for b in batches]))
            for c in range(len(batches[0]))]


def hash_np(batches, groups: Sequence[int], vcols: Sequence[int]) -> Dict[tuple, List]:
    cols = _concat(batches)
    n = len(cols[0][0])
    gid, keys = ax.group_of_rows(cols, groups)
    ng = len(keys)
    first = np.full(ng, n, dtype=np.int64)
    np.minimum.at(first, gid, np.arange(n, dtype=np.int64))
    per = []
    for v in vcols:
        nl, bits = _nulls(cols[v]), value_bits(cols[v][0])
        if ng == 1:
            nn = np.flatnonzero(~nl)
            per.append([int(bits[nn[0]]) if len(nn) else None])
        else:
            per.append([None if nl[r] else int(bits[r]) for r in first.tolist()])
    return {tuple(keys[g]): [p[g] for p in per] for g in range(ng)}


def sorted_literal(cols, groups: Sequence[int], vcols: Sequence[int]) -> List[Tuple[tuple, List]]:
    """-> [(first row's key bits, [first non-NULL value per column])] in input order (itertools.groupby over run ids)."""
    n = len(cols[0][0]) if cols else 0
    ids = sref.run_ids(cols, groups)
    out = []
    for _, rows in itertools.groupby(range(n), key=lambda r: ids[r]):
        rows = list(rows)
        key = tuple(_value(cols[g], rows[0]) for g in groups)
        vals = []
        for v in vcols:
            vals.append(next((_value(cols[v], r) for r in rows if _value(cols[v], r) is not None), None))
        out.append((key, vals))
    return out


def sorted_np(cols, groups: Sequence[int], vcols: Sequence[int]) -> List[Tuple[tuple, List]]:
    n = len(cols[0][0]) if cols else 0
    if n == 0:
        return []
    ids = sref.run_ids_np(cols, groups)
    ng = int(ids[-1]) + 1
    heads = np.flatnonzero(np.r_[True, ids[1:] != ids[:-1]])
    keys = [[None if _nulls(cols[g])[h] else int(value_bits(cols[g][0])[h]) for h in heads.tolist()] for g in groups]
    per = []
    for v in vcols:
        nl, bits = _nulls(cols[v]), value_bits(cols[v][0])
        first = np.full(ng, n, dtype=np.int64)
        ok = np.flatnonzero(~nl)
        np.minimum.at(first, ids[ok], ok)
        per.append([None if f == n else int(bits[f]) for f in first.tolist()])
    return [(tuple(k[g] for k in keys), [p[g] for p in per]) for g in range(ng)]


def output_values(col) -> List[Optional[int]]:
    """A result column as None / value bits."""
    d, nl = col
    d = np.asarray(d)
    nl = np.zeros(len(d), bool) if nl is None else np.asarray(nl, bool)
    bits = value_bits(d).tolist()
    return [None if nl[r] else bits[r] for r in range(len(d))]


def hash_output(out_cols, nkeys: int, vcols_at: Sequence[int]) -> Dict[tuple, List]:
    """A gsql_agg result as {canonical key: [value bits of the columns at vcols_at]}; a key seen twice is an error."""
    n = len(out_cols[0][0]) if out_cols else 0
    keys = []
    for c in range(nkeys):
        d, nl = out_cols[c]
        nl = np.zeros(n, bool) if nl is None else np.asarray(nl, bool)
        img = ax._key_image(np.asarray(d), nl).tolist()
        keys.append([None if nl[r] else img[r] for r in range(n)])
    vals = [output_values(out_cols[c]) for c in vcols_at]
    out = {}
    for r in range(n):
        k = tuple(kc[r] for kc in keys)
        assert k not in out, f"group {k} appears twice"
        out[k] = [v[r] for v in vals]
    return out


def sorted_output(out_cols, nkeys: int, vcols_at: Sequence[int]) -> List[Tuple[tuple, List]]:
    n = len(out_cols[0][0]) if out_cols else 0
    keys = [output_values(out_cols[c]) for c in range(nkeys)]
    vals = [output_values(out_cols[c]) for c in vcols_at]
    return [(tuple(k[r] for k in keys), [v[r] for v in vals]) for r in range(n)]
