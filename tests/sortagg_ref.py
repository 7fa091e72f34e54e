"""Restatement of the reference's SortAggExec (EX/operator/SortAggExec.java:72-135), for checking gsql_sortagg:

  * rows are walked in input order; a row starts a new group when any group key differs from the current group's key
    under NumberType.compare (sort_ref.value_compare != 0): two NULLs are equal, -0.0 and +0.0 differ, every NaN is equal;
  * no group keys: the whole input is one group; empty input: no group at all (currentKey stays null);
  * the key written is the group's first row's, bit for bit; groups come out in input order;
  * aggregates are computed with agg_exact's exact machinery, one group per run.

`run_ids` is the literal walk; `run_ids_np` the same rule over numpy arrays for large inputs.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from tests import agg_exact as ax
from tests import sort_ref as sr


def _type(d) -> int:
    return {np.dtype(np.int32): sr.T_INT32, np.dtype(np.int64): sr.T_INT64, np.dtype(np.float64): sr.T_FP64}[np.asarray(d).dtype]


def run_ids(cols, groups: Sequence[int]) -> np.ndarray:
    """Literal walk (SortAggExec.doNextChunk / checkKeyEqual): the group number of every row."""
    rows = sr.rows_of([cols[g] for g in groups]) if groups else [()] * (len(cols[0][0]) if cols else 0)
    types = [_type(cols[g][0]) for g in groups]
    out, cur, gid = [], None, -1
    for row in rows:
        if cur is None or any(sr.value_compare(a, b, t) != 0 for a, b, t in zip(cur, row, types)):
            gid += 1
            cur = row
        out.append(gid)
    return np.asarray(out, dtype=np.int64)


def _images(d, nl) -> Tuple[np.ndarray, np.ndarray]:
    """(NULL flags, value images equal exactly when NumberType.compare says equal)."""
    d = np.asarray(d)
    isnull = np.zeros(len(d), bool) if nl is None else np.asarray(nl).astype(bool)
    if d.dtype == np.float64:
        img = d.view(np.int64).copy()
        img[np.isnan(d)] = 0x7FF8000000000000  # Double.doubleToLongBits
    else:
        img = d.astype(np.int64)
    img[isnull] = 0
    return isnull, img


def run_ids_np(cols, groups: Sequence[int]) -> np.ndarray:
    n = len(cols[0][0]) if cols else 0
    head = np.zeros(n, bool)
    if n:
        head[0] = True
    for g in groups:
        isnull, img = _images(*cols[g])
        head[1:] |= (isnull[1:] != isnull[:-1]) | (img[1:] != img[:-1])
    return np.cumsum(head) - 1


class SortAggRef:
    """The reference's output for `cols`: `keys[c]` = (values, nulls) of group key c (the first rows'), `ref` = an
    agg_exact.Reference whose single group key is the run number."""

    def __init__(self, cols, groups: Sequence[int], aggs: Sequence[Tuple[int, Sequence[int]]], literal: bool = False):
        rid = run_ids(cols, groups) if literal else run_ids_np(cols, groups)
        n = len(rid)
        self.ngroups = int(rid[-1]) + 1 if n else 0
        first = np.flatnonzero(np.r_[True, rid[1:] != rid[:-1]]) if n else np.zeros(0, np.int64)
        self.first = first
        self.keys = []
        for g in groups:
            d, nl = cols[g]
            self.keys.append((np.asarray(d)[first], None if nl is None else np.asarray(nl).astype(bool)[first]))
        self.run = rid
        self.ref = ax.Reference(list(cols) + [(rid, None)], [len(cols)], aggs) if n else None
        self.aggs = aggs

    def closed_before(self, rows: int) -> int:
        """Groups complete once the first `rows` rows were consumed: all but the one the last of them belongs to."""
        return 0 if rows == 0 else int(self.run[rows - 1])


def compare(got_cols, want: SortAggRef, mode: str = "exact", term_roundings=None):
    """Row for row, in order: keys bit for bit (NULL flags and raw bits), aggregates as agg_exact.compare checks them."""
    nk = len(want.keys)
    n = len(got_cols[0][0]) if got_cols else 0
    assert n == want.ngroups, f"{n} groups, want {want.ngroups}"
    for c in range(nk):
        gd, gn = got_cols[c]
        wd, wn = want.keys[c]
        gnull = np.zeros(n, bool) if gn is None else np.asarray(gn).astype(bool)
        wnull = np.zeros(n, bool) if wn is None else wn
        assert np.array_equal(gnull, wnull), f"key {c}: NULL flags differ"
        gb = np.asarray(gd).astype(np.int64) if np.asarray(gd).dtype == np.int32 else np.asarray(gd).view(np.int64)
        wb = np.asarray(wd).astype(np.int64) if np.asarray(wd).dtype == np.int32 else np.asarray(wd).view(np.int64)
        bad = np.flatnonzero(~wnull & (gb != wb))
        assert not len(bad), f"key {c}: rows {bad[:8].tolist()} differ: got {gb[bad[:4]]}, want {wb[bad[:4]]}"
    if n == 0 or not want.aggs:
        return
    vals = []
    for d, nl in got_cols[nk:]:
        d = np.asarray(d)
        if d.ndim == 2:  # DEC128 (lo, hi) -> Python ints
            d = np.array([(int(h) << 64) + int(lo) for lo, h in zip(d[:, 0].astype(np.uint64).tolist(), d[:, 1].tolist())], dtype=object)
        vals.append((d, nl))
    ax.compare([(np.arange(n, dtype=np.int64), None)] + vals, want.ref, mode, term_roundings)


def concat(parts: Sequence[Sequence[Tuple[np.ndarray, Optional[np.ndarray]]]]) -> List[Tuple[np.ndarray, Optional[np.ndarray]]]:
    """Output batches (lists of (values, nulls)) -> one list of columns."""
    parts = [p for p in parts if p and len(p[0][0])]
    if not parts:
        return []
    out = []
    for c in range(len(parts[0])):
        d = np.concatenate([np.asarray(p[c][0]) for p in parts])
        nl = np.concatenate([np.zeros(len(p[c][0]), bool) if p[c][1] is None else np.asarray(p[c][1]).astype(bool) for p in parts])
        out.append((d, nl))
    return out
