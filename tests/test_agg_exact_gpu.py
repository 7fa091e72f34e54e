"""Every group-by front end against the exact reference of tests/agg_exact.py.

Floating SUM / AVG are compared bit for bit on dyadic data (exact in any summation order) and within the rigorous
gamma_(n-1) * sum|x| bound on ordinary decimal data; COUNT, SUM0 and the 128-bit SUM(INT / BIGINT) as integers; DOUBLE
MIN / MAX by bit pattern.  Each case forces its kernel with the switches gsql_agg_consume reads and asserts from the
context's kernel profile that the kernel ran, so that a change to kernel selection cannot silently drop coverage.
Each case feeds several batches: a 1-row batch, one that is not a multiple of any tile, and a ragged rest.
"""
import functools
import math
import sys

import numpy as np
import pytest

from tests import agg_exact as ax
from tests import kat_util as ku

pytestmark = pytest.mark.gpu

PRIVATE = {"agg_reg", "agg_lane", "agg_smem", "agg_consume"}


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


def _N():
    from galaxysql_b200 import native as N
    return N


def run_agg(gu, cols, types, groups, aggs, edges, expected_groups=64, derived=(), row_filter=None, misaligned=False,
            filter_args=None, host=False):
    """Device batches [edges[i], edges[i+1]) through one HashAgg handle -> (numpy result, DEC128 as Python ints; profile).
    host: numpy (host) batches instead."""
    import torch
    from galaxysql_b200 import api
    N = _N()
    ctx = gu.ctx()
    ctx.profile(True)
    ctx.profile_reset()
    a = api.HashAgg(ctx, types, groups, aggs, expected_groups, filter_args=filter_args, derived=derived, row_filter=row_filter)
    keep = []
    for lo, hi in zip(edges[:-1], edges[1:]):
        if hi <= lo:
            continue
        if host:
            a.consume([(np.ascontiguousarray(d[lo:hi]), None if nl is None else np.ascontiguousarray(nl[lo:hi]).astype(np.uint8))
                       for d, nl in cols])
            continue
        batch = []
        for d, nl in cols:
            if misaligned:  # one leading element: the view starts 4 or 8 bytes off a 16-byte boundary
                t = torch.from_numpy(np.concatenate([d[:1], d[lo:hi]])).cuda()
                keep.append(t)
                assert t[1:].data_ptr() % 16 != 0
                t = t[1:]
            else:
                t = torch.from_numpy(np.ascontiguousarray(d[lo:hi])).cuda()
            tn = None if nl is None else torch.from_numpy(np.ascontiguousarray(nl[lo:hi]).astype(np.uint8)).cuda()
            batch.append((t, tn))
        a.consume(batch)
    res = a.result(N.MEM_DEVICE)
    out = []
    for (d, nl), t in zip(res, a.out_types):
        d, nl = d.cpu().numpy(), nl.cpu().numpy().astype(bool)
        if t == N.T_DEC128:
            d = np.array(api.dec128_to_int(d), dtype=object)
        out.append((d, nl))
    a.close()
    prof = ctx.profile_dump()
    ctx.profile(False)
    return out, prof


def edges_for(n, tile=1024):
    """A 1-row batch, a batch of tile-1 rows (not a multiple of any tile), a large batch and a ragged rest."""
    return [0, 1, tile, tile + (n - tile) // 2, n]


# switches per front end: (environment, the profile name of the kernel that must run)
FRONTS = {
    "reg_pipe": ({}, "agg_reg"),                                             # k_agg_reg_pipe (aligned columns)
    "reg_misaligned": ({}, "agg_reg"),                                       # k_agg_reg, per-thread cp.async (off 16 B)
    "reg_three_stages": ({"GSQL_AGG_REG_STAGES": "3"}, "agg_reg"),
    "lane": ({"GSQL_AGG_NO_REG": "1"}, "agg_lane"),
    "smem": ({"GSQL_AGG_NO_REG": "1", "GSQL_AGG_NO_LANE": "1"}, "agg_smem"),
    "generic": ({"GSQL_AGG_NO_REG": "1", "GSQL_AGG_NO_FAST": "1"}, "agg_consume"),
}


def force(monkeypatch, front):
    env, name = FRONTS[front]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return name


# ------------------------------------------------------------------------------------------------ Q1 shape, dyadic
Q1_N = 1_200_007
Q1_CUTOFF = 10471


@functools.lru_cache(maxsize=None)
def q1_dyadic(ngroups):
    """TPC-H Q1 shape on dyadic data: qty = m/4 and price = p/4 with mixed signs, disc = j/64 (j in [0, 10]), tax = t/64
    (t in [0, 8]); price*(1-disc) = p(64-j)/2^8 and price*(1-disc)*(1+tax) = p(64-j)(64+t)/2^14 are exact.  With >= 6
    groups, every row of group 5 fails the row filter."""
    N = _N()
    n = Q1_N
    g = (ku.rand_u64(n, 101) % np.uint64(ngroups)).astype(np.int64)
    flag, status = (g // 2 - 3).astype(np.int32), (g % 2).astype(np.int32)
    qty, _ = ax.dyadic(ax.dyadic_numerators(n, 102), 2)
    pm = ax.dyadic_numerators(n, 103, big=1 << 34)
    price, _ = ax.dyadic(pm, 2)
    j = (ku.rand_u64(n, 104) % np.uint64(11)).astype(np.int64)
    t = (ku.rand_u64(n, 105) % np.uint64(9)).astype(np.int64)
    disc, tax = np.ldexp(j.astype(np.float64), -6), np.ldexp(t.astype(np.float64), -6)
    e1n, e2n = pm * (64 - j), pm * (64 - j) * (64 + t)
    ax.assert_dyadic_bound(e2n)
    e1, e2 = price * (1.0 - disc), price * (1.0 - disc) * (1.0 + tax)
    assert np.array_equal(e1, np.ldexp(e1n.astype(np.float64), -8)) and np.array_equal(e2, np.ldexp(e2n.astype(np.float64), -14))
    ship = ((ku.rand_u64(n, 106) % np.uint64(2526)) + np.uint64(8036)).astype(np.int32)
    ship[g == 5] = Q1_CUTOFF + 1 + (ship[g == 5] % 50)
    cols = [(flag, None), (status, None), (qty, None), (price, None), (disc, None), (tax, None), (ship, None)]
    types = [N.T_INT32, N.T_INT32, N.T_FP64, N.T_FP64, N.T_FP64, N.T_FP64, N.T_INT32]
    derived = [(N.EXPR_MUL_1MINUS, 3, 4, 0), (N.EXPR_MUL_1MINUS_1PLUS, 3, 4, 5)]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_SUM, [3]), (N.AGG_SUM, [7]), (N.AGG_SUM, [8]), (N.AGG_AVG, [2]), (N.AGG_AVG, [3]),
            (N.AGG_AVG, [4]), (N.AGG_COUNT_STAR, [])]
    ref = ax.Reference(cols + [(e1, None), (e2, None)], [0, 1], aggs, row_mask=ship <= Q1_CUTOFF)
    return cols, types, derived, aggs, ref


Q1_CASES = [(f, 6) for f in FRONTS] + [(f, g) for f in ("reg_pipe", "lane", "smem", "generic") for g in (1, 13, 40)]


@pytest.mark.parametrize("front,ngroups", Q1_CASES, ids=[f"{f}-{g}" for f, g in Q1_CASES])
def test_q1_shape_dyadic_sums_bit_exact(gu, monkeypatch, front, ngroups):
    """Plain and both fused derived sums, AVG, COUNT(*) and the row filter: every SUM / AVG equal to the exact value."""
    N = _N()
    name = force(monkeypatch, front)
    cols, types, derived, aggs, ref = q1_dyadic(ngroups)
    got, prof = run_agg(gu, cols, types, [0, 1], aggs, edges_for(Q1_N), expected_groups=64, derived=derived,
                        row_filter=(6, N.CMP_LE, Q1_CUTOFF), misaligned=front == "reg_misaligned")
    assert name in prof, prof
    if ngroups <= 6 or front == "generic":
        assert PRIVATE & set(prof) == {name}, prof
    if ngroups == 40 and front in ("reg_pipe", "lane"):   # in-kernel fallback, then another kernel on the later batches
        assert len(PRIVATE & set(prof)) >= 2, prof
    if ngroups >= 6:
        assert (-1, 1) not in ax.result_by_key(got, 2)      # every row of group 5 fails the filter: no row, not COUNT 0
    ax.compare(got, ref, mode="exact")


# ------------------------------------------------------------------------------------------------ Q1 shape, decimal data
@functools.lru_cache(maxsize=None)
def q1_decimal():
    N = _N()
    n = Q1_N
    g = (ku.rand_u64(n, 201) % np.uint64(6)).astype(np.int64)
    flag, status = (g // 2).astype(np.int32), (g % 2).astype(np.int32)
    qty = ((ku.rand_u64(n, 202) % np.uint64(50)) + np.uint64(1)).astype(np.float64)
    price = ((ku.rand_u64(n, 203) % np.uint64(10_410_000)) + np.uint64(90_000)).astype(np.float64) / 100.0
    disc = (ku.rand_u64(n, 204) % np.uint64(11)).astype(np.float64) / 100.0
    tax = (ku.rand_u64(n, 205) % np.uint64(9)).astype(np.float64) / 100.0
    ship = ((ku.rand_u64(n, 206) % np.uint64(2526)) + np.uint64(8036)).astype(np.int32)
    cols = [(flag, None), (status, None), (qty, None), (price, None), (disc, None), (tax, None), (ship, None)]
    types = [N.T_INT32, N.T_INT32, N.T_FP64, N.T_FP64, N.T_FP64, N.T_FP64, N.T_INT32]
    derived = [(N.EXPR_MUL_1MINUS, 3, 4, 0), (N.EXPR_MUL_1MINUS_1PLUS, 3, 4, 5)]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_SUM, [3]), (N.AGG_SUM, [7]), (N.AGG_SUM, [8]), (N.AGG_AVG, [3]), (N.AGG_AVG, [4]),
            (N.AGG_COUNT_STAR, [])]
    e1 = price * (1.0 - disc)
    e2 = e1 * (1.0 + tax)
    ref = ax.Reference(cols + [(e1, None), (e2, None)], [0, 1], aggs, row_mask=ship <= Q1_CUTOFF)
    return cols, types, derived, aggs, ref


@pytest.mark.parametrize("front", ["reg_pipe", "lane", "smem", "generic"])
def test_q1_shape_decimal_sums_within_the_gamma_bound(gu, monkeypatch, front):
    """Ordinary decimal data (price / 100, disc / 100): every SUM within gamma_(n-1) * sum|x| of the exact sum, AVG within
    that over n plus one rounding of the division — about 1e-10 relative here, not 1e-6.  The derived sums allow two
    more roundings per term: a fused multiply-add may skip the rounding of the product numpy applied."""
    N = _N()
    name = force(monkeypatch, front)
    cols, types, derived, aggs, ref = q1_decimal()
    got, prof = run_agg(gu, cols, types, [0, 1], aggs, edges_for(Q1_N), derived=derived, row_filter=(6, N.CMP_LE, Q1_CUTOFF))
    assert PRIVATE & set(prof) == {name}, prof
    ax.compare(got, ref, mode="bound", term_roundings={2: 2, 3: 2})


# ------------------------------------------------------------------------------------------------ generic shape
GEN_N = 900_001


@functools.lru_cache(maxsize=None)
def generic_shape(four_keys):
    """Nullable INT key x DOUBLE key (-0.0 / +0.0 as one key, NaNs of both signs as one key): 6 groups.  Group 3's
    measure is NULL in every row; group 4's is NULL in every row of the first three batches and has values in the last."""
    N = _N()
    n = GEN_N
    g = (ku.rand_u64(n, 301) % np.uint64(6)).astype(np.int64)
    r = np.arange(n)
    k1 = np.zeros(n, np.int32)
    k1n = g % 2 == 1
    k1[k1n] = (r[k1n] % 7).astype(np.int32)                      # values under a NULL flag are unspecified
    kd = np.where(g // 2 == 0, np.where(r % 2 == 0, 0.0, -0.0), np.where(g // 2 == 1, 2.5, np.where(r % 3 == 0, -np.nan, np.nan)))
    v, _ = ax.dyadic(ax.dyadic_numerators(n, 302, big=1 << 40), 3)
    vn = (ku.rand_u64(n, 303) % np.uint64(20)) == 0
    vn |= g == 3
    vn |= (g == 4) & (r < edges_for(n)[3])
    w = ku.rand_u64(n, 304).view(np.int64).copy()
    wn = (ku.rand_u64(n, 305) % np.uint64(25)) == 0
    cols = [(k1, k1n), (kd, None), (v, vn), (w, wn)]
    types = [N.T_INT32, N.T_FP64, N.T_FP64, N.T_INT64]
    groups = [0, 1]
    if four_keys:
        cols += [((g % 2 * 1_000_000_007).astype(np.int64) << 20, None), ((g // 2).astype(np.int32), None)]
        types += [N.T_INT64, N.T_INT32]
        groups = [0, 1, 4, 5]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [2]), (N.AGG_COUNT, [2, 3]), (N.AGG_SUM, [2]), (N.AGG_AVG, [2]),
            (N.AGG_SUM0, [3]), (N.AGG_MIN, [2]), (N.AGG_MAX, [2])]
    ref = ax.Reference(cols, groups, aggs)
    assert len(ref.groups) == 6
    return cols, types, groups, aggs, ref


@pytest.mark.parametrize("front", ["lane", "smem", "generic", "generic_four_keys"])
def test_generic_shape_dyadic_and_null_states(gu, monkeypatch, front):
    """COUNT(x), COUNT(x, y), SUM, AVG, SUM0, MIN, MAX with NULL keys and values: exact, and NULL SUM / AVG / MIN / MAX,
    COUNT(x) = 0 for the all-NULL group; the group whose first value arrives in the last batch is not NULL."""
    name = force(monkeypatch, "generic" if front == "generic_four_keys" else front)
    cols, types, groups, aggs, ref = generic_shape(front == "generic_four_keys")
    got, prof = run_agg(gu, cols, types, groups, aggs, edges_for(GEN_N))
    assert PRIVATE & set(prof) == {name}, prof
    ax.compare(got, ref, mode="exact")
    rows = ax.result_by_key(got, len(groups))
    nulls = [k for k, vals in rows.items() if vals[1] == 0]
    assert len(nulls) == 1 and rows[nulls[0]][3:5] == [None, None] and rows[nulls[0]][6:] == [None, None]


# ------------------------------------------------------------------------------------------------ high cardinality
@pytest.mark.parametrize("front", ["prepass_scalar", "prepass_split", "grow"])
def test_high_cardinality_paths_exact(gu, monkeypatch, front):
    """The slot-range pre-pass (scalar scatter with NULL masks; the split kernels for one NULL-free BIGINT key) and the
    re-run of overflowed rows after a table grow.  BIGINT keys sit just above 2^60: adjacent keys tie as float64."""
    N = _N()
    n = 1_000_003
    k = (ku.rand_u64(n, 401) % np.uint64(150_000)).astype(np.int64) + np.int64(1 << 60)
    v, _ = ax.dyadic(ax.dyadic_numerators(n, 402, big=1 << 36), 4)
    w = ku.rand_u64(n, 403).view(np.int64).copy()
    if front == "prepass_split":
        cols, types = [(k, None), (v, None)], [N.T_INT64, N.T_FP64]
        aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [1]), (N.AGG_AVG, [1]), (N.AGG_MIN, [1])]
    else:
        cols = [ku.with_nulls(k, 0.01, 404), ku.with_nulls(v, 0.05, 405), (w, None)]
        types = [N.T_INT64, N.T_FP64, N.T_INT64]
        aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [1]), (N.AGG_AVG, [1]), (N.AGG_MAX, [1]), (N.AGG_SUM, [2]), (N.AGG_SUM0, [2])]
    if front.startswith("prepass"):
        monkeypatch.setenv("GSQL_AGG_PARTITION_MIN_ROWS", "1000")
        monkeypatch.setenv("GSQL_AGG_PARTITION_BYTES", str((4 << 20) if front == "prepass_split" else (1 << 20)))
        expected = 300_000
    else:
        expected = 16
    got, prof = run_agg(gu, cols, types, [0], aggs, edges_for(n), expected_groups=expected)
    assert "agg_consume" in prof, prof
    assert ("agg_rehash" if front == "grow" else "agg_part_scatter") in prof, prof
    ax.compare(got, ax.Reference(cols, [0], aggs), mode="exact")


# ------------------------------------------------------------------------------------------------ two-phase AVG
@pytest.mark.parametrize("mode", ["partial", "shuffle", "avg_merge"])
def test_two_phase_avg_bit_exact(gu, mode):
    """TwoPhaseAgg on one rank (partial: SUM + COUNT partials merged by AVG_MERGE; shuffle: raw rows) and a direct
    AVG_MERGE handle: on dyadic data the merged AVG is the correctly rounded S / n."""
    from galaxysql_b200 import pipelines
    N = _N()
    n = 400_003
    k = ku.with_nulls((ku.rand_u64(n, 501) % np.uint64(40)).astype(np.int64) - 20, 0.01, 502)
    v = ku.with_nulls(ax.dyadic(ax.dyadic_numerators(n, 503, big=1 << 38), 5)[0], 0.05, 504)
    if mode == "avg_merge":
        cnt = ku.with_nulls((ku.rand_u64(n, 505) % np.uint64(1000)).astype(np.int64), 0.02, 506)
        cols = [k, v, cnt]
        aggs = [(N.AGG_AVG_MERGE, [1, 2])]
        got, prof = run_agg(gu, cols, [N.T_INT64, N.T_FP64, N.T_INT64], [0], aggs, edges_for(n))
        assert "agg_consume" in prof, prof
        ax.compare(got, ax.Reference(cols, [0], aggs), mode="exact")
        return
    calls = [(N.AGG_AVG, [1]), (N.AGG_SUM, [1]), (N.AGG_COUNT, [1]), (N.AGG_COUNT_STAR, [])]
    agg = pipelines.TwoPhaseAgg(gu.ctx(), [N.T_INT64, N.T_FP64], [0], calls, expected_groups=64, capacity=n, mode=mode,
                                nslabs=3, nullable=[0, 1])
    out = gu.to_numpy(agg.run(gu.to_device([k, v])))
    agg.close()
    ax.compare(out, ax.Reference([k, v], [0], calls), mode="exact")


# ------------------------------------------------------------------------------------------------ DOUBLE MIN / MAX
DBL_MAX = sys.float_info.max


@pytest.mark.parametrize("front", ["lane", "smem", "generic"])
def test_double_min_max_special_values(gu, monkeypatch, front):
    """NaN, -0.0 / +0.0 in both orders, +-Inf, subnormals and +-DBL_MAX placed so that competing values sit in different
    lanes, warps, CTAs and batches: the per-row path and every merge decide some result.  Compared by bit pattern."""
    N = _N()
    name = force(monkeypatch, front)
    n = 600_001
    g = (ku.rand_u64(n, 601) % np.uint64(8)).astype(np.int32)
    m = ax.dyadic_numerators(n, 602, tiny=1000, nbig=0)
    x = np.ldexp(np.where(m == 0, 1, m).astype(np.float64), -2)           # non-zero finite background
    rows = [np.flatnonzero(g == i) for i in range(8)]
    x[rows[0][-5]] = np.nan                                                # one NaN, in the last batch
    x[rows[1]] = np.where(np.arange(len(rows[1])) % 2 == 0, 0.0, -0.0)     # only zeros, both signs everywhere
    x[rows[2][len(rows[2]) // 3]] = np.inf                                 # +Inf in one batch, -Inf in another
    x[rows[2][-2]] = -np.inf
    x[rows[3]] = np.where(np.arange(len(rows[3])) % 3 == 0, -5e-324, np.where(np.arange(len(rows[3])) % 3 == 1, 5e-324, -0.0))
    x[rows[4][7]], x[rows[4][-7]] = DBL_MAX, -DBL_MAX
    x[rows[5]] = np.abs(x[rows[5]])
    x[rows[5][100]], x[rows[5][-100]] = -0.0, 0.0                          # MIN -0.0 over positives and +0.0
    x[rows[6]] = -0.0
    x[rows[6][-1]] = 0.0                                                   # a single +0.0 in the last row of the group
    x[rows[7]] = 0.0
    x[rows[7][len(rows[7]) // 2]] = -0.0                                   # a single -0.0 mid-table (another CTA)
    cols = [(g, None), (x, None)]
    aggs = [(N.AGG_MIN, [1]), (N.AGG_MAX, [1]), (N.AGG_COUNT_STAR, [])]
    got, prof = run_agg(gu, cols, [N.T_INT32, N.T_FP64], [0], aggs, edges_for(n))
    assert PRIVATE & set(prof) == {name}, prof
    ref = ax.Reference(cols, [0], aggs)
    assert math.isnan(ref.groups[(0,)][0]) and ax.f64_bits(ref.groups[(1,)][0]) == ax.f64_bits(-0.0)
    assert ax.f64_bits(ref.groups[(6,)][1]) == ax.f64_bits(0.0) and ax.f64_bits(ref.groups[(7,)][0]) == ax.f64_bits(-0.0)
    ax.compare(got, ref)


# ------------------------------------------------------------------------------------------------ Inf / NaN in sums
@pytest.mark.parametrize("front", ["reg_pipe", "lane", "smem", "generic"])
def test_non_finite_sums_stay_in_their_group(gu, monkeypatch, front):
    """+Inf, NaN, Inf - Inf and -Inf in another column land in their own groups only; a row that the row filter rejects
    holds +Inf and must not change any group.  Every other group stays exact."""
    N = _N()
    name = force(monkeypatch, front)
    n = 700_001
    g = (ku.rand_u64(n, 701) % np.uint64(6)).astype(np.int64)
    flag, status = (g // 2).astype(np.int32), (g % 2).astype(np.int32)
    qty, _ = ax.dyadic(ax.dyadic_numerators(n, 702), 2)
    price, _ = ax.dyadic(ax.dyadic_numerators(n, 703, big=1 << 34), 2)
    ship = ((ku.rand_u64(n, 704) % np.uint64(2526)) + np.uint64(8036)).astype(np.int32)
    keep = ship <= Q1_CUTOFF
    rows = [np.flatnonzero((g == i) & keep) for i in range(6)]
    price[rows[0][[5, len(rows[0]) // 2, -3]]] = np.inf
    price[rows[1][7]] = np.nan
    price[rows[2][11]], price[rows[2][-11]] = np.inf, -np.inf
    qty[rows[3][3]] = -np.inf
    price[np.flatnonzero((g == 4) & ~keep)[[0, -1]]] = np.inf                # rejected by the filter
    cols = [(flag, None), (status, None), (qty, None), (price, None), (ship, None)]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_SUM, [3]), (N.AGG_AVG, [3]), (N.AGG_COUNT_STAR, [])]
    got, prof = run_agg(gu, cols, [N.T_INT32, N.T_INT32, N.T_FP64, N.T_FP64, N.T_INT32], [0, 1], aggs, edges_for(n),
                        row_filter=(4, N.CMP_LE, Q1_CUTOFF))
    assert PRIVATE & set(prof) == {name}, prof
    ref = ax.Reference(cols, [0, 1], aggs, row_mask=keep)
    assert ref.groups[(0, 0)][1].value == math.inf and math.isnan(ref.groups[(0, 1)][1].value)
    assert math.isnan(ref.groups[(1, 0)][1].value) and ref.groups[(1, 1)][0].value == -math.inf
    assert ref.groups[(2, 0)][1].special is None and ref.groups[(2, 0)][2].special is None
    ax.compare(got, ref, mode="exact")


# ------------------------------------------------------------------------------------------------ SUM(BIGINT / INT)
@pytest.mark.parametrize("variant", ["one_batch", "many_batches", "nulls_many_batches", "prepass", "grow"])
def test_sum_bigint_exact_across_2_pow_64(gu, monkeypatch, variant):
    """128-bit SUM(BIGINT) and SUM(INT), SUM0's wraparound, integer MIN / MAX: values at and near +-2^63 (INT64_MIN
    included) whose group totals cross +-2^64 many times in both directions; compared with Python integers."""
    N = _N()
    big_groups = variant == "grow"
    n = 800_011
    ng = 100_000 if big_groups else 7
    k = (ku.rand_u64(n, 801) % np.uint64(ng)).astype(np.int64) - 3
    w = ku.rand_u64(n, 802).view(np.int64).copy()
    ext = np.array([ax.INT64_MIN, ax.INT64_MIN + 1, ax.INT64_MAX, ax.INT64_MAX - 1, -1, 1], dtype=np.int64)
    pick = ku.rand_u64(n, 803) % np.uint64(4) == 0
    w[pick] = ext[(ku.rand_u64(n, 804) % np.uint64(6)).astype(np.int64)[pick]]
    w[k == -3] = ax.INT64_MIN                                   # one group of INT64_MIN only: total -n * 2^63
    w[k == -2] = ax.INT64_MAX
    i32 = ku.rand_u64(n, 805).view(np.int64).astype(np.int32)
    i32[:2] = [-(1 << 31), (1 << 31) - 1]
    wn = ((ku.rand_u64(n, 806) % np.uint64(10)) == 0) if variant in ("nulls_many_batches", "prepass") else None
    cols = [(k, None), (w, wn), (i32, None)]
    aggs = [(N.AGG_SUM, [1]), (N.AGG_SUM, [2]), (N.AGG_SUM0, [1]), (N.AGG_COUNT, [1]), (N.AGG_MIN, [1]), (N.AGG_MAX, [1]),
            (N.AGG_COUNT_STAR, [])]
    if variant == "prepass":
        monkeypatch.setenv("GSQL_AGG_PARTITION_MIN_ROWS", "1000")
        monkeypatch.setenv("GSQL_AGG_PARTITION_BYTES", str(1 << 20))
    edges = [0, n] if variant == "one_batch" else (list(np.linspace(0, n, 38).astype(int)) if "many" in variant else edges_for(n))
    got, prof = run_agg(gu, cols, [N.T_INT64, N.T_INT64, N.T_INT32], [0], aggs, edges, expected_groups=16)
    assert "agg_consume" in prof, prof
    if variant == "prepass":
        assert "agg_part_scatter" in prof, prof
    if variant == "grow":
        assert "agg_rehash" in prof, prof
    ref = ax.Reference(cols, [0], aggs)
    if not big_groups:
        sums = [vals[0] for vals in ref.groups.values()]
        assert max(sums) > (1 << 64) and min(sums) < -(1 << 64)
    ax.compare(got, ref)


# ------------------------------------------------------------------------------------------------ row filter
@pytest.mark.parametrize("front", ["reg_pipe", "lane", "smem", "generic"])
def test_row_filter_boundaries(gu, monkeypatch, front):
    """Every comparison against the filter column's minimum and maximum, and LT INT64_MIN / GT INT64_MAX on a BIGINT
    column (the register plan rewrites them as empty intervals): the surviving groups' sums bit for bit, and a group
    whose every row fails is absent."""
    N = _N()
    name = force(monkeypatch, front)
    n = 100_003
    g = (ku.rand_u64(n, 901) % np.uint64(5)).astype(np.int64)
    flag, status = (g // 2).astype(np.int32), (g % 2).astype(np.int32)
    price, _ = ax.dyadic(ax.dyadic_numerators(n, 902, big=1 << 34), 2)
    f64 = ku.rand_u64(n, 903).view(np.int64).copy()
    f64[g == 0] &= np.int64(-2)                                 # even in group 0, odd in group 4
    f64[g == 4] |= np.int64(1)
    f64[[10, n - 10]] = [ax.INT64_MIN, ax.INT64_MAX]
    f32 = (ku.rand_u64(n, 904) % np.uint64(1000)).astype(np.int32) - 500
    cols = [(flag, None), (status, None), (price, None), (f64, None), (f32, None)]
    types = [N.T_INT32, N.T_INT32, N.T_FP64, N.T_INT64, N.T_INT32]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_AVG, [2]), (N.AGG_COUNT_STAR, [])]
    ops = {N.CMP_LE: np.less_equal, N.CMP_LT: np.less, N.CMP_GE: np.greater_equal, N.CMP_GT: np.greater,
           N.CMP_EQ: np.equal, N.CMP_NE: np.not_equal}
    cases = [(3, op, c) for op in ops for c in (ax.INT64_MIN, ax.INT64_MAX)]
    cases += [(4, op, c) for op in ops for c in (int(f32.min()), int(f32.max()))]
    cases += [(3, N.CMP_EQ, int(f64[g == 0][3]))]               # one row of group 0 passes
    for col, op, c in cases:
        mask = ops[op](cols[col][0].astype(np.int64), c)
        got, prof = run_agg(gu, cols, types, [0, 1], aggs, edges_for(n), row_filter=(col, op, c))
        assert PRIVATE & set(prof) == {name}, (col, op, c, prof)
        ref = ax.Reference(cols, [0, 1], aggs, row_mask=mask)
        if col == 3 and op == N.CMP_EQ:
            assert len(ref.groups) == 1, (c, ref.groups)           # every other group is absent, not COUNT(*) = 0
        ax.compare(got, ref, mode="exact")
