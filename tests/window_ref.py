"""Restatement of NonFrameOverWindowExec (EX/operator/NonFrameOverWindowExec.java:79-146) with RowNumber, Rank, DenseRank
and the running aggregates, row by row as the stock loop runs them.  Shares no code with the product.

`window_rows(batches, partition, calls, reset)`:
  batches    list of batches, each a list of (values, nulls-or-None) numpy columns
  partition  partition column indexes
  calls      (kind, columns) with kind a name: ROW_NUMBER, RANK, DENSE_RANK, COUNT_STAR, COUNT, SUM, SUM0, AVG, MIN, MAX
  reset      the CURRENT ROW .. CURRENT ROW frame: one flag for every call, or one per call (resetAccumulators)
-> one list per call of the values written to every row (None = NULL): Python ints for the rank family, counts, SUM0 and
   SUM over integers (the DECIMAL sum), floats for DOUBLE results.

DOUBLE SUM / AVG add in row order from the first value, as LittleNum2DoubleSum does; `exact=True` gives the exact prefix sum
(a Fraction) instead, for error bounds.  MIN / MAX follow Math.min / Math.max: NaN wins, -0.0 < +0.0.

`window_np` is an independent vectorised definition of ROW_NUMBER / RANK / DENSE_RANK / COUNT(*) / SUM over integers for
input whose partitions are contiguous, used at sizes the row loop cannot reach.
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction

import numpy as np


def _bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]


def obj_equals(a, b) -> bool:
    """Object.equals / Objects.equals on Integer, Long and Double boxes: Double by doubleToLongBits."""
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, float):
        if math.isnan(a) and math.isnan(b):
            return True
        return _bits(a) == _bits(b)
    return a == b


def _obj(col, r):
    vals, nulls = col
    if nulls is not None and nulls[r]:
        return None
    v = vals[r]
    return float(v) if vals.dtype == np.float64 else int(v)


def _wrap64(v: int) -> int:
    return (v + (1 << 63)) % (1 << 64) - (1 << 63)


def _jmin(a: float, b: float) -> float:
    if math.isnan(a) or math.isnan(b):
        return math.nan
    if a == b == 0.0:
        return a if math.copysign(1, a) < 0 else b
    return a if a < b else b


def _jmax(a: float, b: float) -> float:
    if math.isnan(a) or math.isnan(b):
        return math.nan
    if a == b == 0.0:
        return a if math.copysign(1, a) > 0 else b
    return a if a > b else b


class _Call:
    def __init__(self, kind, cols, exact):
        self.kind, self.cols, self.exact = kind, list(cols), exact
        self.reset()

    def reset(self):  # resetToInitValue
        self.n = 0          # RowNumber.number, Rank.count
        self.rank = 0
        self.last = None    # Rank.lastRow (its peer values), None = no row yet
        self.v = None       # aggregate value, None = NULL
        self.cnt = 0

    def accumulate(self, row):
        k = self.kind
        if k == "ROW_NUMBER":
            self.n += 1
        elif k in ("RANK", "DENSE_RANK"):
            peer = tuple(row[c] for c in self.cols)
            same = self.last is not None and all(obj_equals(a, b) for a, b in zip(self.last, peer))
            if k == "RANK":
                self.n += 1
                if not same:
                    self.rank, self.last = self.n, peer
            elif not same:
                self.rank += 1
                self.last = peer
        elif k == "COUNT_STAR":
            self.cnt += 1
        elif k == "COUNT":
            if all(row[c] is not None for c in self.cols):
                self.cnt += 1
        else:
            x = row[self.cols[0]]
            if k == "SUM0":
                self.v = _wrap64((self.v or 0) + (x if x is not None else 0))
                return
            if x is None:
                return
            if k in ("SUM", "AVG"):
                if isinstance(x, float) and self.exact:
                    x = Fraction(x) if math.isfinite(x) else x
                self.v = x if self.v is None else self.v + x
                self.cnt += 1
            elif k == "MIN":
                self.v = x if self.v is None else (_jmin(self.v, x) if isinstance(x, float) else min(self.v, x))
            elif k == "MAX":
                self.v = x if self.v is None else (_jmax(self.v, x) if isinstance(x, float) else max(self.v, x))

    def result(self):  # writeResultTo
        k = self.kind
        if k == "ROW_NUMBER":
            return self.n
        if k in ("RANK", "DENSE_RANK"):
            return self.rank
        if k in ("COUNT_STAR", "COUNT"):
            return self.cnt
        if k == "SUM0":
            return self.v or 0
        if k == "AVG":
            return None if self.v is None else self.v / self.cnt
        return self.v


def window_rows(batches, partition, calls, reset=False, exact=False):
    resets = list(reset) if isinstance(reset, (list, tuple)) else [reset] * len(calls)
    st = [_Call(k, c, exact) for k, c in calls]
    out = [[] for _ in calls]
    last_part = None  # lastPartition (its partition values)
    first = True
    for cols in batches:
        n = len(cols[0][0]) if cols else 0
        for r in range(n):
            row = [_obj(c, r) for c in cols]
            part = tuple(row[c] for c in partition)
            change = first or not all(obj_equals(a, b) for a, b in zip(last_part, part))
            first = False
            if change:
                last_part = part
            for i, s in enumerate(st):
                if resets[i] or change:
                    s.reset()
                s.accumulate(row)
                out[i].append(s.result())
    return out


def window_np(cols, partition, calls):
    """Vectorised definition for partitions that are contiguous runs: heads where any partition column (NULL flag or
    value) changes; peers likewise on a call's columns.  Integer and NULL-free DOUBLE columns only (DOUBLE compared by
    value, so no ±0.0 or NaN)."""
    n = len(cols[0][0])
    idx = np.arange(n, dtype=np.int64)

    def changes(which):
        h = np.zeros(n, dtype=bool)
        h[0] = True
        for c in which:
            v, nl = cols[c]
            h[1:] |= v[1:] != v[:-1]
            if nl is not None:
                nl = nl.astype(bool)
                h[1:] |= nl[1:] != nl[:-1]
        return h

    head = changes(partition)
    start = np.maximum.accumulate(np.where(head, idx, 0))
    out = []
    for kind, cc in calls:
        if kind == "ROW_NUMBER" or kind == "COUNT_STAR":
            out.append(idx - start + 1)
        elif kind in ("RANK", "DENSE_RANK"):
            peer = head | changes(cc)
            if kind == "RANK":
                out.append(np.maximum.accumulate(np.where(peer, idx, 0)) - start + 1)
            else:
                c = np.cumsum(peer)
                out.append(c - c[start] + 1)
        elif kind == "SUM":  # integer input, no NULLs, |prefix| < 2^63
            v = cols[cc[0]][0].astype(np.int64)
            c = np.cumsum(v)
            out.append(c - c[start] + v[start])
        else:
            raise ValueError(kind)
    return out
