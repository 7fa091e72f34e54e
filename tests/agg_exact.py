"""Exact references for the group-by's aggregates (tests only): plain numpy and Python integers, independent of the C oracle.

* Dyadic columns (`m * 2^-k`, integer m) whose absolute numerators sum below 2^53: every partial sum of such a column is
  an fp64 number, so every summation order and tree gives the same, exact result.  The kernels' SUM and AVG must then
  match the reference bit for bit.
* Other data: a floating sum computed by any tree of pairwise additions satisfies |got - S| <= gamma_(n-1) * sum|x|
  (gamma_k = k*u / (1 - k*u), u = 2^-53), which `sum_error_bound` evaluates in exact rational arithmetic.
* Group results are keyed on exact images (Python ints, canonical double bits), never on keys cast to float64.

Semantics restated here (DESIGN §2): DOUBLE group keys -0.0 / +0.0 are one key and every NaN is one key; MIN / MAX
follow Java's Math.min / Math.max (NaN wins, -0.0 < +0.0); SUM(INT / BIGINT) is exact; SUM0 wraps like a Java long;
SUM, AVG, MIN, MAX of a group without a non-NULL value are NULL.  A zero floating SUM / AVG compares equal whatever its
sign: the kernels' accumulators start at +0.0.
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from galaxysql_b200 import native as N
from tests import kat_util as ku

U = Fraction(1, 1 << 53)
NAN_KEY = 0x7FF8000000000000  # the one image of every NaN group key
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1

Col = Tuple[np.ndarray, Optional[np.ndarray]]


# ------------------------------------------------------------------------------------------------ scalars
def f64_bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", float(x)))[0]


def java_min(a: float, b: float) -> float:
    """java.lang.Math.min(double, double)."""
    if a != a:
        return a
    if b != b:
        return b
    if a == 0.0 and b == 0.0:
        return a if math.copysign(1.0, a) < 0 else b
    return a if a < b else b


def java_max(a: float, b: float) -> float:
    """java.lang.Math.max(double, double)."""
    if a != a:
        return a
    if b != b:
        return b
    if a == 0.0 and b == 0.0:
        return b if math.copysign(1.0, a) < 0 else a
    return a if a > b else b


def java_fold(values, is_max: bool) -> float:
    f = java_max if is_max else java_min
    it = iter(values)
    acc = next(it)
    for v in it:
        acc = f(v, acc)
    return acc


def wrap_i64(s: int) -> int:
    """A Python int as the Java long it wraps to."""
    s &= (1 << 64) - 1
    return s - (1 << 64) if s >> 63 else s


def gamma(k: int) -> Fraction:
    return k * U / (1 - k * U)


def sum_error_bound(n: int, abs_sum: Fraction, term_roundings: int = 0) -> Fraction:
    """Largest |computed - exact| of a sum of n terms over any order / tree of additions, where abs_sum = sum|x_i|.
    term_roundings > 0 when the kernel may form each term with that many roundings of its own that the x_i passed to the
    reference did not see (a fused multiply-add into the accumulator skips the product's rounding)."""
    if n <= 1 and term_roundings == 0:
        return Fraction(0)
    r = term_roundings
    if r == 0:
        return gamma(n - 1) * abs_sum
    return (gamma(n - 1 + r) + gamma(r)) / (1 - gamma(r)) * abs_sum


# ------------------------------------------------------------------------------------------------ generators
def exact_int_sum(v: np.ndarray) -> int:
    """Exact sum of an int64 array (up to ~2^31 rows), without int64 overflow."""
    v = np.asarray(v, dtype=np.int64)
    return (int((v >> np.int64(32)).sum()) << 32) + int((v & np.int64(0xFFFFFFFF)).sum())


def assert_dyadic_bound(*numerators: np.ndarray) -> int:
    """The absolute numerators of a column (or of several columns summed as one) stay below 2^53: then every partial
    sum over any subset of rows is exact in fp64.  Returns the bound's value."""
    total = 0
    for m in numerators:
        m = np.asarray(m, dtype=np.int64)
        assert int(np.abs(m).max(initial=0)) < (1 << 53)
        total += exact_int_sum(np.abs(m))
    assert total < (1 << 53), f"sum of |numerators| = 2^{math.log2(max(total, 1)):.2f} >= 2^53: sums would round"
    return total


def dyadic_numerators(n: int, seed: int, tiny: int = 3, mid: int = 1 << 15, mid_every: int = 10, big: int = 1 << 30,
                      nbig: int = 8) -> np.ndarray:
    """Mixed-sign integer numerators: most rows tiny (|m| <= tiny), every mid_every-th row up to `mid`, and `nbig` rows
    near `big` — large-magnitude values next to many small ones, heavy cancellation within every group."""
    r = ku.rand_u64(n, seed)
    mag = (r >> np.uint64(8)) % np.uint64(tiny + 1)
    sel = (r & np.uint64(0xFF)) % np.uint64(mid_every) == 0
    mag = np.where(sel, (r >> np.uint64(20)) % np.uint64(mid), mag).astype(np.int64)
    m = np.where((r >> np.uint64(63)) == 1, -mag, mag)
    if nbig and n:
        at = (ku.rand_u64(nbig, seed + 7777) % np.uint64(n)).astype(np.int64)
        m[at] = np.where(np.arange(nbig) % 2 == 0, big - np.arange(nbig), -(big - 3 * np.arange(nbig)))
    return m.astype(np.int64)


def dyadic(m: np.ndarray, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """(float64 column m * 2^-k, numerators); asserts the column's sums are exact in any order."""
    m = np.asarray(m, dtype=np.int64)
    assert_dyadic_bound(m)
    return np.ldexp(m.astype(np.float64), -k), m


# ------------------------------------------------------------------------------------------------ exact sums of doubles
def _scaled(x: np.ndarray):
    """Finite float64 values -> (numerators, K) with x == numerator * 2^-K exactly.  Numerators are int64 when every
    one of them and every group sum fits (the common case), else Python ints in an object array."""
    num = np.zeros(len(x), dtype=np.int64)
    nz = x != 0
    if not nz.any():
        return num, 0
    mf, e = np.frexp(x[nz])
    M = (mf * 2.0 ** 53).astype(np.int64)           # exact: |mf| in [0.5, 1)
    E = e.astype(np.int64) - 53
    low = M & -M                                     # lowest set bit: strip the trailing zeros
    tz = np.frexp(low.astype(np.float64))[1].astype(np.int64) - 1
    M >>= tz
    E += tz
    K = max(0, int(-E.min()))
    sh = E + K
    bits = np.frexp(np.abs(M).astype(np.float64))[1].astype(np.int64) + sh
    if int(bits.max()) <= 61:
        num[nz] = M << sh
        return num, K
    out = np.zeros(len(x), dtype=object)
    out[np.flatnonzero(nz)] = [int(a) << int(s) for a, s in zip(M.tolist(), sh.tolist())]
    return out, K


def _group_int_sums(v: np.ndarray, gid: np.ndarray, ngroups: int) -> List[int]:
    """Exact per-group sums of int64 (or Python-int object) values."""
    if v.dtype == object:
        out = [0] * ngroups
        for g, x in zip(gid.tolist(), v.tolist()):
            out[g] += x
        return out
    hi = np.zeros(ngroups, dtype=np.int64)
    lo = np.zeros(ngroups, dtype=np.int64)
    np.add.at(hi, gid, v >> np.int64(32))
    np.add.at(lo, gid, v & np.int64(0xFFFFFFFF))
    return [(int(h) << 32) + int(l) for h, l in zip(hi.tolist(), lo.tolist())]


class ExactSum:
    """Floating SUM (avg=False) or AVG of one group: the exact sum S of its values, sum|x|, the number of values, or a
    non-finite result (Inf / NaN, order-independent)."""
    __slots__ = ("S", "A", "n", "special", "avg")

    def __init__(self, S: Fraction, A: Fraction, n: int, special: Optional[float], avg: bool):
        self.S, self.A, self.n, self.special, self.avg = S, A, n, special, avg

    @property
    def value(self) -> float:
        if self.special is not None:
            return self.special
        return float(self.S / self.n) if self.avg else float(self.S)

    def __repr__(self):
        return f"ExactSum({'avg' if self.avg else 'sum'}={self.value!r}, n={self.n})"


# ------------------------------------------------------------------------------------------------ the group reference
def _key_image(d: np.ndarray, nl: np.ndarray) -> np.ndarray:
    d = np.asarray(d)
    if d.dtype == np.float64:
        img = d.view(np.int64).copy()
        img[d == 0] = 0                    # -0.0 and +0.0: one key
        img[np.isnan(d)] = NAN_KEY         # every NaN: one key
    else:
        img = d.astype(np.int64)
    img[nl] = 0
    return img


def _nulls(c: Col) -> np.ndarray:
    d, nl = c
    return np.zeros(len(d), bool) if nl is None else np.asarray(nl, bool)


def group_of_rows(cols: Sequence[Col], groups: Sequence[int]):
    """-> (gid per row, list of exact key tuples by gid).  A key component is None (NULL), a Python int (INT / BIGINT)
    or the canonical bit image of a DOUBLE."""
    n = len(cols[0][0]) if cols else 0
    if not groups:
        return np.zeros(n, dtype=np.int64), [()]
    code = np.zeros(n, dtype=np.int64)
    for c in groups:
        nl = _nulls(cols[c])
        for part in (nl.astype(np.int64), _key_image(cols[c][0], nl)):
            u, inv = np.unique(part, return_inverse=True)
            code = np.unique(code * len(u) + inv.reshape(-1), return_inverse=True)[1].reshape(-1).astype(np.int64)
    ng = int(code.max()) + 1 if n else 0
    first = np.full(ng, n, dtype=np.int64)
    np.minimum.at(first, code, np.arange(n, dtype=np.int64))
    comps = []
    for c in groups:
        nl = _nulls(cols[c])[first].tolist()
        img = _key_image(np.asarray(cols[c][0])[first], np.zeros(ng, bool)).tolist()
        comps.append([None if z else v for z, v in zip(nl, img)])
    return code, list(zip(*comps))


def _float_sums(x: np.ndarray, ok: np.ndarray, gid: np.ndarray, ng: int, avg: bool) -> List[Optional[ExactSum]]:
    cnt = np.bincount(gid[ok], minlength=ng)
    xv = np.where(ok, x, 0.0)
    nan = np.bincount(gid, weights=(ok & np.isnan(x)).astype(np.float64), minlength=ng) > 0
    pinf = np.bincount(gid, weights=(ok & (x == np.inf)).astype(np.float64), minlength=ng) > 0
    ninf = np.bincount(gid, weights=(ok & (x == -np.inf)).astype(np.float64), minlength=ng) > 0
    xv = np.where(np.isfinite(xv), xv, 0.0)
    num, K = _scaled(xv)
    S = _group_int_sums(num, gid, ng)
    A = _group_int_sums(np.abs(num) if num.dtype != object else np.array([abs(v) for v in num.tolist()], dtype=object), gid, ng)
    out: List[Optional[ExactSum]] = []
    for g in range(ng):
        if cnt[g] == 0:
            out.append(None)
            continue
        special = None
        if nan[g] or (pinf[g] and ninf[g]):
            special = math.nan
        elif pinf[g]:
            special = math.inf
        elif ninf[g]:
            special = -math.inf
        out.append(ExactSum(Fraction(S[g], 1 << K), Fraction(A[g], 1 << K), int(cnt[g]), special, avg))
    return out


def _float_minmax(x: np.ndarray, ok: np.ndarray, gid: np.ndarray, ng: int, is_max: bool) -> List[Optional[float]]:
    """Java fold per group.  The fold runs over a candidate set that provably contains the result — one NaN, the
    smallest / largest non-zero non-NaN value (an unambiguous numeric order) and each sign of zero present — because a
    Java min / max fold does not depend on the order of its operands (up to the NaN payload)."""
    cnt = np.bincount(gid[ok], minlength=ng)
    isnan = ok & np.isnan(x)
    nz = ok & ~np.isnan(x) & (x != 0)
    negz = ok & (x == 0) & np.signbit(x)
    posz = ok & (x == 0) & ~np.signbit(x)
    ext = np.full(ng, -np.inf if is_max else np.inf)
    (np.maximum if is_max else np.minimum).at(ext, gid[nz], x[nz])
    has = [np.bincount(gid[m], minlength=ng) > 0 for m in (isnan, nz, negz, posz)]
    out: List[Optional[float]] = []
    for g in range(ng):
        if cnt[g] == 0:
            out.append(None)
            continue
        cand = []
        if has[0][g]:
            cand.append(math.nan)
        if has[1][g]:
            cand.append(float(ext[g]))
        if has[2][g]:
            cand.append(-0.0)
        if has[3][g]:
            cand.append(0.0)
        out.append(java_fold(cand, is_max))
    return out


class Reference:
    """Exact GROUP BY result: `groups` maps the exact key tuple to the list of aggregate values (see module doc)."""

    def __init__(self, cols: Sequence[Col], groups: Sequence[int], aggs: Sequence[Tuple[int, Sequence[int]]],
                 row_mask: Optional[np.ndarray] = None):
        if row_mask is not None:
            cols = [(np.asarray(d)[row_mask], None if nl is None else np.asarray(nl, bool)[row_mask]) for d, nl in cols]
        self.key_types = [_type_of(cols[c][0]) for c in groups]
        self.kinds = [k for k, _ in aggs]
        self.in_types = [_type_of(cols[c[0]][0]) if c else N.T_INT64 for _, c in aggs]
        gid, keys = group_of_rows(cols, groups)
        ng = len(keys)
        per_agg = []
        for kind, ac in aggs:
            ac = list(ac)
            if kind == N.AGG_COUNT_STAR:
                per_agg.append([int(v) for v in np.bincount(gid, minlength=ng)])
                continue
            ok = ~_nulls(cols[ac[0]])
            for c in ac[1:]:
                if kind == N.AGG_COUNT:
                    ok = ok & ~_nulls(cols[c])
            if kind == N.AGG_COUNT:
                per_agg.append([int(v) for v in np.bincount(gid[ok], minlength=ng)])
                continue
            x = np.asarray(cols[ac[0]][0])
            cnt = np.bincount(gid[ok], minlength=ng)
            if kind in (N.AGG_SUM, N.AGG_AVG) and x.dtype == np.float64:
                per_agg.append(_float_sums(x, ok, gid, ng, kind == N.AGG_AVG))
            elif kind == N.AGG_AVG_MERGE:   # (partial sum, partial count): NULL partial sums are skipped
                s = _float_sums(x, ok, gid, ng, False)
                cn = cols[ac[1]]
                okc = ok & ~_nulls(cn)
                tot = _group_int_sums(np.where(okc, np.asarray(cn[0], np.int64), 0), gid, ng)
                res = []
                for g in range(ng):
                    if s[g] is None or tot[g] == 0:
                        res.append(None)
                    else:
                        res.append(ExactSum(s[g].S, s[g].A, tot[g], s[g].special, True))
                per_agg.append(res)
            elif kind in (N.AGG_SUM, N.AGG_SUM0):
                S = _group_int_sums(np.where(ok, x.astype(np.int64), 0), gid, ng)
                if kind == N.AGG_SUM0:
                    per_agg.append([wrap_i64(s) for s in S])
                else:
                    per_agg.append([S[g] if cnt[g] else None for g in range(ng)])
            elif kind in (N.AGG_MIN, N.AGG_MAX) and x.dtype == np.float64:
                per_agg.append(_float_minmax(x, ok, gid, ng, kind == N.AGG_MAX))
            elif kind in (N.AGG_MIN, N.AGG_MAX):
                ext = np.full(ng, INT64_MIN if kind == N.AGG_MAX else INT64_MAX, dtype=np.int64)
                (np.maximum if kind == N.AGG_MAX else np.minimum).at(ext, gid[ok], x[ok].astype(np.int64))
                per_agg.append([int(ext[g]) if cnt[g] else None for g in range(ng)])
            else:
                raise ValueError(f"aggregate kind {kind} over {x.dtype}")
        self.groups: Dict[tuple, list] = {keys[g]: [a[g] for a in per_agg] for g in range(ng)}


def _type_of(d) -> int:
    return {np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}[np.asarray(d).dtype]


# ------------------------------------------------------------------------------------------------ comparator
def result_by_key(cols: Sequence[Col], nkeys: int) -> Dict[tuple, list]:
    """A group-by result (keys first, then one column per aggregate; DEC128 as Python ints) keyed on exact key images.
    A key that appears twice is an error."""
    n = len(cols[0][0]) if cols else 0
    keys = []
    for c in range(nkeys):
        d, nl = cols[c]
        nl = np.zeros(n, bool) if nl is None else np.asarray(nl, bool)
        img = _key_image(np.asarray(d), nl).tolist()
        keys.append([None if nl[r] else img[r] for r in range(n)])
    vals = []
    for c in range(nkeys, len(cols)):
        d, nl = cols[c]
        nl = np.zeros(n, bool) if nl is None else np.asarray(nl, bool)
        dl = np.asarray(d).tolist()
        vals.append([None if nl[r] else dl[r] for r in range(n)])
    out: Dict[tuple, list] = {}
    for r in range(n):
        k = tuple(keys[c][r] for c in range(nkeys))
        assert k not in out, f"group {k} appears twice in the result"
        out[k] = [v[r] for v in vals]
    return out


def _float_eq_special(got: float, want: float) -> bool:
    if math.isnan(want):
        return math.isnan(got)
    return got == want


def compare(got_cols: Sequence[Col], ref: Reference, mode: str = "exact", term_roundings: Optional[Dict[int, int]] = None,
            max_report: int = 12) -> None:
    """Asserts that a group-by result equals the reference.  Integers (COUNT, SUM0, SUM(INT) as DEC128, integer
    MIN / MAX) exactly; DOUBLE MIN / MAX by bit pattern (any NaN matches any NaN); floating SUM / AVG with `==` against
    the exact value (mode "exact", dyadic inputs: a zero matches either sign) or within `sum_error_bound` (mode "bound")."""
    nk = len(ref.key_types)
    got = result_by_key(got_cols, nk)
    bad = []
    missing = [k for k in ref.groups if k not in got]
    extra = [k for k in got if k not in ref.groups]
    if missing or extra:
        bad.append(f"groups missing {missing[:8]} ({len(missing)}), unexpected {extra[:8]} ({len(extra)})")
    tr = term_roundings or {}
    for k, want_row in ref.groups.items():
        if k not in got:
            continue
        for a, (want, g) in enumerate(zip(want_row, got[k])):
            kind, it = ref.kinds[a], ref.in_types[a]
            ok = True
            if want is None or g is None:
                ok = want is None and g is None
            elif isinstance(want, ExactSum):
                if want.special is not None or not math.isfinite(g):
                    ok = _float_eq_special(g, want.value)
                elif mode == "exact":
                    ok = (Fraction(g) == want.S) if not want.avg else (g == want.value)
                else:
                    err = sum_error_bound(want.n, want.A, tr.get(a, 0))
                    if want.avg:
                        ok = abs(Fraction(g) - want.S / want.n) <= err / want.n + U * abs(Fraction(g))
                    else:
                        ok = abs(Fraction(g) - want.S) <= err
            elif kind in (N.AGG_MIN, N.AGG_MAX) and it == N.T_FP64:
                ok = (math.isnan(g) and math.isnan(want)) or f64_bits(g) == f64_bits(want)
            else:
                ok = int(g) == want and not isinstance(g, float)
            if not ok:
                bad.append(f"group {k} aggregate {a} (kind {kind}): got {g!r}, want {want!r}")
    assert not bad, f"{len(bad)} mismatches:\n  " + "\n  ".join(bad[:max_report])
