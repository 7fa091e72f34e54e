"""The hash aggregation's per-aggregate FILTER argument (gsql_agg_call.filter_arg, AggregateCall.filterArg) on every path
that takes it, against the exact reference of tests/agg_exact.py.

The rule (AggOpenHashMap.putChunk): a row is left out of one aggregate only when that aggregate's filter cell is a
non-NULL BIGINT below 1; INT and DOUBLE cells and NULLs never filter, and the row's group is created before the filter is
looked at, so a group whose every row fails a call's filter still exists (COUNT 0, SUM / AVG / MIN / MAX NULL, SUM0 0).
The kernels apply it in accumulate() (the generic row loop, the shared-memory kernel's in-kernel fallback, the re-run
of overflowed rows) and twice in k_agg_smem (the fused fp64 SUM / AVG reduction and the per-aggregate loop); the lane and
register front ends refuse a spec with a FILTER.  Every aggregation case asserts from the kernel profile which kernels
ran.
Floating data is dyadic, so every SUM / AVG is compared bit for bit.
"""
import functools

import numpy as np
import pytest

from tests import agg_exact as ax
from tests import kat_util as ku
from tests.test_agg_exact_gpu import PRIVATE, edges_for, force, run_agg

pytestmark = pytest.mark.gpu

FSPEC = np.array([ax.INT64_MIN, -1, 0, 1, 2, ax.INT64_MAX], dtype=np.int64)


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


def _N():
    from galaxysql_b200 import native as N
    return N


def _front(monkeypatch, front):
    """"default": no switches; otherwise test_agg_exact_gpu's FRONTS."""
    return None if front == "default" else force(monkeypatch, front)


def _types(cols):
    N = _N()
    return [{np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}[d.dtype]
            for d, _ in cols]


# ------------------------------------------------------------------------------------------------ filter columns
def f_i64(n, seed, null_frac=0.15):
    """BIGINT filter: INT64_MIN, -1, 0, 1, 2, INT64_MAX and NULLs, drawn row by row (mixed within every warp)."""
    return ku.with_nulls(FSPEC[(ku.rand_u64(n, seed) % np.uint64(len(FSPEC))).astype(np.int64)], null_frac, seed + 1)


def f_i32(n, seed):
    """INT filter with 0 and negative values: never filters."""
    return (ku.rand_u64(n, seed) % np.uint64(5)).astype(np.int32) - np.int32(3), None


def f_f64(n, seed, null_frac=0.0):
    """DOUBLE filter with 0.0, -0.0, -1.0 and NaN: never filters."""
    return ku.with_nulls(np.array([0.0, -1.0, np.nan, -0.0, 2.0])[(ku.rand_u64(n, seed) % np.uint64(5)).astype(np.int64)],
                         null_frac, seed + 1)


def dyadic_col(n, seed, k=3, null_frac=0.0, big=1 << 36):
    return ku.with_nulls(ax.dyadic(ax.dyadic_numerators(n, seed, big=big), k)[0], null_frac, seed + 1)


def check(got, cols, groups, aggs, filter_args, row_mask=None):
    ref = ax.Reference(cols, groups, aggs, row_mask=row_mask, filter_args=filter_args)
    ax.compare(got, ref, mode="exact")
    return ref


# ------------------------------------------------------------------------------------------------ selection
@functools.lru_cache(maxsize=None)
def q1_filtered():
    """Q1-like: two INT keys, 6 groups, fp64 SUMs and AVG; f is a BIGINT FILTER that rejects every row of group 4."""
    n = 1_000_003
    g = (ku.rand_u64(n, 1001) % np.uint64(6)).astype(np.int64)
    flag, status = (g // 2).astype(np.int32), (g % 2).astype(np.int32)
    qty, price = dyadic_col(n, 1002, 2), dyadic_col(n, 1004, 2, big=1 << 34)
    f, fn = f_i64(n, 1006)
    f, fn = f.copy(), fn.copy()
    f[g == 4], fn[g == 4] = 0, False
    return [(flag, None), (status, None), qty, price, (f, fn)]


def test_filter_takes_the_smem_kernel_and_the_plain_spec_the_register_one(gu, monkeypatch):
    """With one FILTER the register and lane front ends refuse the spec and the shared-memory kernel runs; the same spec
    without the FILTER takes the register kernel, so the profile assertion is known to bite."""
    N = _N()
    cols = q1_filtered()
    aggs = [(N.AGG_SUM, [2]), (N.AGG_SUM, [3]), (N.AGG_AVG, [2]), (N.AGG_COUNT_STAR, [])]
    fa = [-1, 4, -1, -1]
    got, prof = run_agg(gu, cols, _types(cols), [0, 1], aggs, edges_for(len(cols[0][0])), filter_args=fa)
    assert PRIVATE & set(prof) == {"agg_smem"}, prof
    ref = check(got, cols, [0, 1], aggs, fa)
    assert ref.groups[(2, 0)][1] is None and ref.groups[(2, 0)][3] > 0
    got, prof = run_agg(gu, cols, _types(cols), [0, 1], aggs, edges_for(len(cols[0][0])))
    assert PRIVATE & set(prof) == {"agg_reg"}, prof
    check(got, cols, [0, 1], aggs, None)


# ------------------------------------------------------------------------------------------------ smem: both filter sites
@functools.lru_cache(maxsize=None)
def wide(ngroups):
    """One INT key, one DOUBLE value and six FILTER columns (8 used columns, AF_MAX_USED): 2-5 BIGINT (4 rejects every
    row of key 0), 6 INT, 7 DOUBLE.  Column 8 is a second INT key for the nine-column case."""
    n = 1_000_003
    k = (ku.rand_u64(n, 1101) % np.uint64(ngroups)).astype(np.int32)
    v = dyadic_col(n, 1102, 3, null_frac=0.05)
    f2, f3, f4, f5 = f_i64(n, 1104), f_i64(n, 1106, 0.0), f_i64(n, 1108, 0.3), f_i64(n, 1110, 0.02)
    f4 = (np.where(k == 0, 0, f4[0]).astype(np.int64), f4[1] & (k != 0))
    k2 = ((ku.rand_u64(n, 1112) % np.uint64(3)).astype(np.int32), None)
    return [(k, None), v, f2, f3, f4, f5, f_i32(n, 1114), f_f64(n, 1116, 0.1), k2]


def wide_aggs():
    """Ten fp64 SUM / AVG (the first 8 reduced together, AF_MAX_FV; the last two per aggregate, both with filters that
    reject rows), then COUNT(*), COUNT(v, f), SUM0, INT MIN and DOUBLE MAX / MIN: 16 calls, every one but one filtered."""
    N = _N()
    S, A = N.AGG_SUM, N.AGG_AVG
    aggs = [(S, [1]), (A, [1]), (S, [1]), (A, [1]), (S, [1]), (A, [1]), (S, [1]), (A, [1]), (S, [1]), (A, [1]),
            (N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [1, 2]), (N.AGG_SUM0, [3]), (N.AGG_MIN, [2]), (N.AGG_MAX, [1]),
            (N.AGG_MIN, [1])]
    fa = [2, 3, 4, 5, 6, 7, -1, 4, 3, 2, 5, 3, 4, 5, 3, 2]
    return aggs, fa


@pytest.mark.parametrize("ngroups", [7, 40])
def test_smem_fused_and_per_aggregate_filters(gu, monkeypatch, ngroups):
    """7 groups fit every warp table; 40 overflow them, so rows take accumulate() inside k_agg_smem and the host switches
    the later batches to the generic kernel."""
    cols = wide(ngroups)[:8]
    aggs, fa = wide_aggs()
    got, prof = run_agg(gu, cols, _types(cols), [0], aggs, edges_for(len(cols[0][0])), filter_args=fa)
    if ngroups == 7:
        assert PRIVATE & set(prof) == {"agg_smem"}, prof
    else:
        assert {"agg_smem", "agg_consume"} <= set(prof), prof
    ref = check(got, cols, [0], aggs, fa)
    g0 = ref.groups[(0,)]
    assert g0[2] is None and g0[7] is None and g0[12] == 0 and g0[6] is not None   # key 0: every row fails column 4


def test_nine_used_columns_take_the_generic_kernel(gu):
    cols = wide(7)
    aggs, fa = wide_aggs()
    got, prof = run_agg(gu, cols, _types(cols), [0, 8], aggs, edges_for(len(cols[0][0])), filter_args=fa)
    assert PRIVATE & set(prof) == {"agg_consume"}, prof
    check(got, cols, [0, 8], aggs, fa)


# ------------------------------------------------------------------------------------------------ generic, 1-5 keys
@functools.lru_cache(maxsize=None)
def generic_table():
    """Keys: DOUBLE with -0.0 / +0.0 and NaNs of both signs; nullable INT; BIGINT beyond 2^60; INT; nullable BIGINT."""
    n = 600_001
    g = (ku.rand_u64(n, 1201) % np.uint64(12)).astype(np.int64)
    r = np.arange(n)
    kd = np.array([0.0, 2.5, np.nan, -7.0])[g % 4]
    kd = np.where((kd == 0) & (r % 2 == 1), -0.0, kd)
    kd = np.where(np.isnan(kd) & (r % 3 == 0), -np.nan, kd)
    k1 = ((g // 4).astype(np.int32), (g == 11) | (g == 3))
    k2 = (np.int64(1 << 60) + (g % 2), None)
    k3 = ((g % 3).astype(np.int32), None)
    k4 = ku.with_nulls(g // 6, 0.1, 1202)
    v = dyadic_col(n, 1203, 4, null_frac=0.05)
    w = ku.with_nulls(ku.rand_u64(n, 1205).view(np.int64).copy(), 0.04, 1206)
    return [(kd, None), k1, k2, k3, k4, v, w, f_i64(n, 1207), f_i32(n, 1209), f_f64(n, 1211, 0.1)]


@pytest.mark.parametrize("nkeys", [1, 2, 3, 5])
def test_generic_kernel_filters_with_1_to_5_keys(gu, monkeypatch, nkeys):
    """k_agg_consume<1..3> and <0> (5 keys): NULL keys, DOUBLE keys with both zeros and NaNs, every aggregate kind
    including the exact 128-bit SUM(BIGINT) under a filter."""
    N = _N()
    name = force(monkeypatch, "generic")
    cols = generic_table()
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [5]), (N.AGG_COUNT, [5, 6]), (N.AGG_SUM, [5]), (N.AGG_AVG, [5]),
            (N.AGG_SUM0, [6]), (N.AGG_MIN, [5]), (N.AGG_MAX, [5]), (N.AGG_SUM, [6]), (N.AGG_MIN, [6]), (N.AGG_MAX, [6]),
            (N.AGG_COUNT_STAR, [])]
    fa = [7, 7, 8, 7, 9, 7, 7, 7, 7, 8, 7, -1]
    groups = list(range(nkeys))
    got, prof = run_agg(gu, cols, _types(cols), groups, aggs, edges_for(len(cols[0][0])), filter_args=fa)
    assert PRIVATE & set(prof) == {name}, prof
    check(got, cols, groups, aggs, fa)


# ------------------------------------------------------------------------------------------------ mid-stream switch
def test_front_end_switch_mid_stream_carries_filtered_states(gu):
    """Two batches of 5 keys (the shared-memory kernel), a batch of over 100 k distinct keys (the kernel's fallback and
    overflow re-run, then the 2^16-group cut-off), and 5 keys again (now the generic kernel): one set of states."""
    N = _N()
    e = [0, 1, 60_000, 120_000, 420_000, 520_000]
    n = e[-1]
    k = (ku.rand_u64(n, 1301) % np.uint64(5)).astype(np.int64)
    k[e[3]:e[4]] = (ku.rand_u64(e[4] - e[3], 1302) % np.uint64(200_000)).astype(np.int64) + 5
    v = dyadic_col(n, 1303, 3, null_frac=0.03)
    w = (ku.rand_u64(n, 1305).view(np.int64) >> np.int64(3), None)
    cols = [(k, None), v, w, f_i64(n, 1306), f_i32(n, 1308), f_f64(n, 1310)]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [1]), (N.AGG_AVG, [1]), (N.AGG_MIN, [1]), (N.AGG_SUM0, [2]),
            (N.AGG_COUNT, [1]), (N.AGG_MAX, [2]), (N.AGG_SUM, [1])]
    fa = [3, 3, 4, 3, 3, -1, 3, 5]
    got, prof = run_agg(gu, cols, _types(cols), [0], aggs, e, filter_args=fa)
    assert {"agg_smem", "agg_consume", "agg_rehash"} <= set(prof), prof
    assert not {"agg_reg", "agg_lane"} & set(prof), prof
    ref = check(got, cols, [0], aggs, fa)
    assert len(ref.groups) > 100_000


# ------------------------------------------------------------------------------------------------ high cardinality
@pytest.mark.parametrize("front", ["smem_grow", "generic_grow", "prepass_scalar", "prepass_split"])
def test_high_cardinality_filters(gu, monkeypatch, front):
    """About 150 k groups: expected_groups=16 through the shared-memory and the generic kernel (overflowed rows re-run
    after a table grow), and the slot-range pre-pass (the scalar scatter with a nullable filter column; the split kernels
    for one NULL-free BIGINT key, a value and a filter)."""
    N = _N()
    n = 1_000_003
    k = (ku.rand_u64(n, 1401) % np.uint64(150_000)).astype(np.int64) + np.int64(1 << 60)
    if front == "prepass_split":
        cols = [(k, None), dyadic_col(n, 1402, 4), f_i64(n, 1404, 0.0)]
        aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [1]), (N.AGG_AVG, [1]), (N.AGG_MIN, [1]), (N.AGG_COUNT_STAR, [])]
        fa = [2, 2, -1, 2, 2]
    else:
        cols = [ku.with_nulls(k, 0.01, 1406), dyadic_col(n, 1402, 4, null_frac=0.05), (ku.rand_u64(n, 1407).view(np.int64), None),
                f_i64(n, 1408), f_f64(n, 1410)]
        aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [1]), (N.AGG_AVG, [1]), (N.AGG_MAX, [1]), (N.AGG_SUM0, [2]),
                (N.AGG_COUNT, [1]), (N.AGG_SUM, [1])]
        fa = [3, 3, 3, 4, 3, -1, 3]
    if front.startswith("prepass"):
        monkeypatch.setenv("GSQL_AGG_PARTITION_MIN_ROWS", "1000")
        monkeypatch.setenv("GSQL_AGG_PARTITION_BYTES", str((4 << 20) if front == "prepass_split" else (1 << 20)))
        expected = 300_000
    else:
        force(monkeypatch, "smem" if front == "smem_grow" else "generic")
        expected = 16
    got, prof = run_agg(gu, cols, _types(cols), [0], aggs, edges_for(n), expected_groups=expected, filter_args=fa)
    assert "agg_consume" in prof, prof
    if front.startswith("prepass"):
        assert "agg_part_scatter" in prof, prof
    else:
        assert "agg_rehash" in prof, prof
    if front == "smem_grow":
        assert "agg_smem" in prof, prof
    check(got, cols, [0], aggs, fa)


# ------------------------------------------------------------------------------------------------ with Filter / Project
@pytest.mark.parametrize("front", ["default", "generic"])
def test_filter_with_row_filter_and_derived_column(gu, monkeypatch, front):
    """The fused row filter and a derived price*(1-disc)*(1+tax) aggregated under a FILTER: group 5, whose rows all fail
    the row filter, is absent; group 4, whose rows all fail only the FILTER, is present with COUNT 0 and NULL sums."""
    N = _N()
    name = _front(monkeypatch, front) or "agg_smem"
    n = 1_000_003
    g = (ku.rand_u64(n, 1501) % np.uint64(6)).astype(np.int64)
    flag, status = (g // 2).astype(np.int32), (g % 2).astype(np.int32)
    qty, _ = ax.dyadic(ax.dyadic_numerators(n, 1502), 2)
    pm = ax.dyadic_numerators(n, 1503, big=1 << 34)
    price, _ = ax.dyadic(pm, 2)
    j = (ku.rand_u64(n, 1504) % np.uint64(11)).astype(np.int64)
    t = (ku.rand_u64(n, 1505) % np.uint64(9)).astype(np.int64)
    disc, tax = np.ldexp(j.astype(np.float64), -6), np.ldexp(t.astype(np.float64), -6)
    ax.assert_dyadic_bound(pm * (64 - j) * (64 + t))
    e1, e2 = price * (1.0 - disc), price * (1.0 - disc) * (1.0 + tax)
    ship = ((ku.rand_u64(n, 1506) % np.uint64(2526)) + np.uint64(8036)).astype(np.int32)
    cutoff = 10471
    ship[g == 5] = cutoff + 1 + (ship[g == 5] % 50)
    f, fn = f_i64(n, 1507)
    f, fn = f.copy(), fn.copy()
    f[g == 4], fn[g == 4] = -1, False
    cols = [(flag, None), (status, None), (qty, None), (price, None), (disc, None), (tax, None), (ship, None), (f, fn)]
    derived = [(N.EXPR_MUL_1MINUS, 3, 4, 0), (N.EXPR_MUL_1MINUS_1PLUS, 3, 4, 5)]
    aggs = [(N.AGG_SUM, [8]), (N.AGG_SUM, [9]), (N.AGG_AVG, [9]), (N.AGG_SUM, [2]), (N.AGG_COUNT_STAR, []),
            (N.AGG_MAX, [9]), (N.AGG_MIN, [8])]
    fa = [7] * len(aggs)
    got, prof = run_agg(gu, cols, _types(cols), [0, 1], aggs, edges_for(n), derived=derived,
                        row_filter=(6, N.CMP_LE, cutoff), filter_args=fa)
    assert PRIVATE & set(prof) == {name}, prof
    rows = ax.result_by_key(got, 2)
    assert (2, 1) not in rows
    assert rows[(2, 0)] == [None, None, None, None, 0, None, None]
    check(got, cols + [(e1, None), (e2, None)], [0, 1], aggs, fa, row_mask=ship <= cutoff)


# ------------------------------------------------------------------------------------------------ aliasing
@pytest.mark.parametrize("front", ["smem", "generic"])
def test_filter_column_is_the_key_and_the_argument(gu, monkeypatch, front):
    """x is the group key, the FILTER of every call and the argument of COUNT / SUM0 / MIN / MAX (and, on the generic
    kernel, SUM(x) FILTER (x)): the groups x <= 0 keep COUNT(*) 0, the NULL group keeps all its rows."""
    N = _N()
    name = force(monkeypatch, front)
    n = 900_001
    x = f_i64(n, 1601, 0.1)
    v = dyadic_col(n, 1603, 3)
    cols = [x, v]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [0]), (N.AGG_SUM0, [0]), (N.AGG_MIN, [0]), (N.AGG_MAX, [0]),
            (N.AGG_SUM, [1]), (N.AGG_AVG, [1])]
    if front == "generic":
        aggs.append((N.AGG_SUM, [0]))
    fa = [0] * len(aggs)
    got, prof = run_agg(gu, cols, _types(cols), [0], aggs, edges_for(n), filter_args=fa)
    assert PRIVATE & set(prof) == {name}, prof
    ref = check(got, cols, [0], aggs, fa)
    for key in (ax.INT64_MIN, -1, 0):
        assert ref.groups[(key,)][:5] == [0, 0, 0, None, None]
    nul = ref.groups[(None,)]
    assert nul[0] == int(x[1].sum()) and nul[1] == 0 and nul[3] is None


# ------------------------------------------------------------------------------------------------ no group keys
@pytest.mark.parametrize("front", ["smem", "generic", "empty"])
def test_no_group_keys_with_rejecting_filters(gu, monkeypatch, front):
    """Without group keys there is exactly one output row: COUNT 0 and NULL SUM / AVG / MAX where the filter rejects every
    row, and for an empty input."""
    N = _N()
    name = force(monkeypatch, "generic" if front == "empty" else front)
    n = 500_001
    rej = FSPEC[:3][(ku.rand_u64(n, 1701) % np.uint64(3)).astype(np.int64)]
    cols = [dyadic_col(n, 1702, 3, null_frac=0.1), (rej, None), f_i32(n, 1704), f_i64(n, 1705), (rej.astype(np.float64), None)]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [0]), (N.AGG_SUM, [0]), (N.AGG_AVG, [0]), (N.AGG_MAX, [0]),
            (N.AGG_COUNT_STAR, []), (N.AGG_SUM, [0]), (N.AGG_MIN, [0]), (N.AGG_COUNT_STAR, [])]
    fa = [1, 1, 1, 1, 1, 2, 3, 4, 3]
    edges = [0] if front == "empty" else edges_for(n)
    got, prof = run_agg(gu, cols, _types(cols), [], aggs, edges, filter_args=fa)
    if front != "empty":
        assert PRIVATE & set(prof) == {name}, prof
    assert len(got[0][0]) == 1
    ref = check(got, [(d[:edges[-1]], None if nl is None else nl[:edges[-1]]) for d, nl in cols], [], aggs, fa)
    assert ref.groups[()][:5] == [0, 0, None, None, None]
    if front != "empty":
        assert ref.groups[()][5] == n and ref.groups[()][6] is not None


# ------------------------------------------------------------------------------------------------ SUM(BIGINT), 128 bits
@pytest.mark.parametrize("mem", ["device", "host"])
def test_exact_bigint_sum_under_a_filter_across_2_pow_64(gu, mem):
    """Values at and near +-2^63: FILTER a keeps the positive ones (and NULL-filtered rows), FILTER b the negative ones,
    so the filter decides which way each group's 128-bit total crosses 2^64; the unfiltered total cancels."""
    N = _N()
    n = 800_011
    k = (ku.rand_u64(n, 1801) % np.uint64(7)).astype(np.int64)
    ext = np.array([ax.INT64_MIN, ax.INT64_MIN + 1, ax.INT64_MAX, ax.INT64_MAX - 1, -1, 1], dtype=np.int64)
    w = ext[(ku.rand_u64(n, 1802) % np.uint64(6)).astype(np.int64)]
    fa_col = ku.with_nulls(np.where(w > 0, 2, np.where(ku.rand_u64(n, 1803) % np.uint64(2) == 0, 0, ax.INT64_MIN)), 0.01, 1804)
    fb_col = (np.where(w < 0, ax.INT64_MAX, -1).astype(np.int64), None)
    i32 = (ku.rand_u64(n, 1805).view(np.int64).astype(np.int32), None)
    cols = [(k, None), (w, None), i32, fa_col, fb_col]
    aggs = [(N.AGG_SUM, [1]), (N.AGG_SUM, [1]), (N.AGG_SUM, [1]), (N.AGG_SUM0, [1]), (N.AGG_COUNT, [1]), (N.AGG_MIN, [1]),
            (N.AGG_MAX, [1]), (N.AGG_SUM, [2]), (N.AGG_COUNT_STAR, [])]
    fa = [3, 4, -1, 3, 3, 4, 3, 4, -1]
    got, prof = run_agg(gu, cols, _types(cols), [0], aggs, edges_for(n), expected_groups=16, filter_args=fa,
                        host=mem == "host")
    assert PRIVATE & set(prof) == {"agg_consume"}, prof
    ref = check(got, cols, [0], aggs, fa)
    for vals in ref.groups.values():
        assert vals[0] > (1 << 64) and vals[1] < -(1 << 64) and abs(vals[2]) < vals[0]


# ------------------------------------------------------------------------------------------------ batch forms
@pytest.mark.parametrize("front", ["default", "generic"])
@pytest.mark.parametrize("form", ["host", "misaligned", "stripped_mask"])
def test_batch_forms(gu, monkeypatch, front, form):
    """Host batches, device views that start off a 16-byte boundary, and a filter column whose all-zero NULL mask the
    library strips (the kernels then take their NULL-free loads)."""
    N = _N()
    name = _front(monkeypatch, front) or "agg_smem"
    n = 500_003
    g = (ku.rand_u64(n, 1901) % np.uint64(9)).astype(np.int64)
    f, fn = f_i64(n, 1902, 0.0 if form == "stripped_mask" else 0.1)
    if form == "stripped_mask":
        fn = np.zeros(n, bool)
    cols = [((g // 3).astype(np.int32), None), ((g % 3).astype(np.int32), None), dyadic_col(n, 1904, 2), (f, fn),
            f_f64(n, 1906)]
    aggs = [(N.AGG_SUM, [2]), (N.AGG_AVG, [2]), (N.AGG_COUNT_STAR, []), (N.AGG_MIN, [2]), (N.AGG_COUNT, [2]),
            (N.AGG_SUM, [2])]
    fa = [3, 3, 3, 3, 4, -1]
    got, prof = run_agg(gu, cols, _types(cols), [0, 1], aggs, edges_for(n), filter_args=fa, host=form == "host",
                        misaligned=form == "misaligned")
    assert PRIVATE & set(prof) == {name}, prof
    check(got, cols, [0, 1], aggs, fa)


# ------------------------------------------------------------------------------------------------ operator interface
def test_operator_interface_filter_args_equal_the_oracle(gu):
    """operators.GpuHashAggExec with CountRow(filterArg=...), Sum(..., filterArg=...) and friends over 1000-row chunks
    equals the oracle's AggOpenHashMap restatement, row for row."""
    from collections import Counter
    from galaxysql_b200 import operators as o
    from oracle import oracle as orc
    n = 20_000
    k = (ku.rand_u64(n, 2001) % np.uint64(50)).astype(np.int32)
    v = (ku.rand_u64(n, 2002) % np.uint64(1000)).astype(np.float64) - 500.0     # integers: exact in any order
    f, fn = f_i64(n, 2003)
    f = f.copy()
    f[k == 7] = 0
    fn = fn & (k != 7)
    types = [o.DataTypes.IntegerType, o.DataTypes.DoubleType, o.DataTypes.LongType]
    chunks = []
    for lo in range(0, n, 1000):
        hi = lo + 1000
        chunks.append(o.Chunk(o.IntegerBlock(k[lo:hi]), o.DoubleBlock(v[lo:hi]), o.LongBlock(f[lo:hi], fn[lo:hi])))
    aggregators = [o.CountRow(filterArg=2), o.Sum(1, False, None, filterArg=2), o.Count([1], False, 2), o.Min(1, filterArg=2),
                   o.Max(1, filterArg=-1), o.Avg(1, False, None, 2)]
    exec_ = o.GpuHashAggExec(types, [0], aggregators, None, 64, o.ExecutionContext(chunk_size=7))
    got = Counter()
    for ch in o.SingleExecTest(exec_, None, chunks).exec().result():
        got.update(ch.rows())
    exp = orc.hash_agg([(k, None), (v, None), (f, fn)], [0],
                       [orc.AggCall(a.kind, list(a.targetIndexes), a.filterArg) for a in aggregators], 64)
    want = Counter(tuple(None if nl is not None and nl[r] else (d[r].item() if hasattr(d[r], "item") else d[r])
                         for d, nl in exp) for r in range(len(exp[0][0])))
    assert got == want
    assert got[(7, 0, None, 0, None, max(v[k == 7]), None)] == 1


# ------------------------------------------------------------------------------------------------ refusals
def test_filter_on_a_derived_or_missing_column_is_invalid(gu):
    """filter_arg >= n_input_cols (a derived column's index, or past every column) is GSQL_E_INVALID at create."""
    from galaxysql_b200 import api
    N = _N()
    types = [N.T_INT32, N.T_FP64, N.T_FP64, N.T_INT64]
    derived = [(N.EXPR_MUL_1MINUS, 1, 2, 0)]
    for fa in (4, 5, 31):
        with pytest.raises(N.GsqlError) as ei:
            api.HashAgg(gu.ctx(), types, [0], [(N.AGG_SUM, [4])], 64, filter_args=[fa], derived=derived)
        assert ei.value.status == N.E_INVALID, fa
    a = api.HashAgg(gu.ctx(), types, [0], [(N.AGG_SUM, [4])], 64, filter_args=[3], derived=derived)
    a.close()
