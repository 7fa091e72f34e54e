"""GSQL_AGG_FIRST_VALUE on the GPU against tests/first_value_ref.py, bit for bit: as a multiset of groups for gsql_agg and
row for row, in order, for gsql_sortagg.  Covers INT / BIGINT / DOUBLE values with NaN payloads, -0.0, +-Inf and
subnormals; 0-5 group keys (every k_agg_consume_fv instantiation); FIRST_VALUE mixed with other aggregates; many consume
calls; host and device batches; table growth with the overflow re-run; no slot-range pre-pass; sorted groups spanning
tiles and batches; the FILTER refusal; TwoPhaseAgg on one rank; the Python operators."""
import struct

import numpy as np
import pytest

from galaxysql_b200 import api, native as N, operators as ops, pipelines
from tests import agg_exact as ax
from tests import first_value_ref as fv
from tests import kat_util as ku
from tests.gpu_util import ctx, to_device, to_numpy

pytestmark = pytest.mark.gpu

TILE = 2048  # SA_TILE of agg_sorted.cuh


def _nan(payload):
    return struct.unpack("<d", struct.pack("<q", 0x7FF0000000000000 | payload))[0]


SPECIAL = np.array([_nan(0x8000000000001), _nan(0x0000000000BEEF), -0.0, 0.0, np.inf, -np.inf, 5e-324, -2.2e-308, 1.5],
                   np.float64)


def values(n, seed, nulls=0.2):
    """An FP64 column of special values and normals, an INT64 column over the full range, an INT32 column."""
    rng = np.random.default_rng(seed)
    x = np.where(rng.random(n) < 0.5, SPECIAL[rng.integers(0, len(SPECIAL), n)], rng.normal(size=n))
    i64 = ku.rand_u64(n, seed).view(np.int64).copy()
    i32 = rng.integers(-2**31, 2**31, n).astype(np.int32)
    return [(x, rng.random(n) < nulls), (i64, rng.random(n) < nulls), (i32, rng.random(n) < nulls)]


def keys(n, nkeys, ngroups, seed):
    """nkeys columns (INT64, INT32, FP64 in turn) whose combination takes about ngroups values; a few NULLs."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, ngroups, n)
    out = []
    for c in range(nkeys):
        t = c % 3
        if t == 0:
            d = (g * 1_000_000_007 + c).astype(np.int64)
        elif t == 1:
            d = (g % 50_000 + c).astype(np.int32)
        else:
            d = np.array([-0.0, 0.0, np.nan, 2.5], np.float64)[g % 4] if ngroups <= 4 else (g / 7.0).astype(np.float64)
        out.append((d, rng.random(n) < 0.01))
    return out


def run_hash(batches, groups, aggs, expected_groups=1024, mem="host", filter_args=None):
    types = [ax._type_of(d) for d, _ in batches[0]]
    c = ctx()
    c.profile(True)
    c.profile_reset()
    a = api.HashAgg(c, types, groups, aggs, expected_groups, filter_args=filter_args)
    try:
        for b in batches:
            a.consume(to_device(b) if mem == "device" else b)
        out = a.result()
    finally:
        a.close()
    prof = c.profile_dump()
    c.profile(False)
    return out, prof


def split(cols, edges):
    return [[(d[a:b], None if nl is None else nl[a:b]) for d, nl in cols] for a, b in zip(edges[:-1], edges[1:])]


def fv_at(groups, aggs):
    return [len(groups) + i for i, (k, _) in enumerate(aggs) if k == N.AGG_FIRST_VALUE]


def check_hash(batches, groups, aggs, **kw):
    out, prof = run_hash(batches, groups, aggs, **kw)
    vcols = [c[0] for k, c in aggs if k == N.AGG_FIRST_VALUE]
    want = fv.hash_np(batches, groups, vcols)
    got = fv.hash_output(out, len(groups), fv_at(groups, aggs))
    assert got == want
    return out, prof


# ------------------------------------------------------------------------------------------------ hash aggregation
@pytest.mark.parametrize("nkeys", [0, 1, 2, 3, 5])
@pytest.mark.parametrize("mem", ["host", "device"])
def test_hash_values_bit_for_bit_for_every_key_count(nkeys, mem):
    n = 300_007
    cols = keys(n, nkeys, 20_000, 10 + nkeys) + values(n, 20 + nkeys)
    aggs = [(N.AGG_FIRST_VALUE, [nkeys]), (N.AGG_FIRST_VALUE, [nkeys + 1]), (N.AGG_FIRST_VALUE, [nkeys + 2])]
    _, prof = check_hash(split(cols, [0, 1, 1000, 150_000, n]), list(range(nkeys)), aggs, mem=mem)
    assert "agg_consume" in prof, prof


def test_hash_mixed_with_other_aggregates():
    n = 200_003
    cols = keys(n, 2, 5_000, 31) + values(n, 32)
    aggs = [(N.AGG_SUM, [2]), (N.AGG_FIRST_VALUE, [2]), (N.AGG_COUNT_STAR, []), (N.AGG_FIRST_VALUE, [3]),
            (N.AGG_MIN, [3]), (N.AGG_MAX, [4]), (N.AGG_COUNT, [4]), (N.AGG_FIRST_VALUE, [4])]
    batches = split(cols, [0, 77, n // 2, n])
    out, _ = check_hash(batches, [0, 1], aggs)
    rest = [i for i, (k, _) in enumerate(aggs) if k != N.AGG_FIRST_VALUE]
    ax.compare(out[:2] + [out[2 + i] for i in rest], ax.Reference(cols, [0, 1], [aggs[i] for i in rest]), mode="bound")


def test_hash_later_consume_calls_never_override():
    """Every key appears in every one of 60 batches; the first batch holds a NULL for a third of the keys."""
    nk, nb = 3000, 60
    batches = []
    for b in range(nb):
        k = np.random.default_rng(b).permutation(nk).astype(np.int64)
        v = (k * 1000 + b).astype(np.int64)
        nl = (k % 3 == 0) if b == 0 else np.zeros(nk, bool)
        batches.append([(k, np.zeros(nk, bool)), (v, nl)])
    out, _ = check_hash(batches, [0], [(N.AGG_FIRST_VALUE, [1])], mem="device")
    got = fv.hash_output(out, 1, [1])
    assert got[(3,)] == [None] and got[(4,)] == [4000]


def test_hash_one_group_rules():
    n = 5000
    v = (np.arange(n) * 3).astype(np.int64)
    nl = np.arange(n) < 1234  # the first 1234 rows are NULL
    k = np.full(n, 9, np.int64)
    for groups, cols in (([0], [(k, np.zeros(n, bool)), (v, nl)]), ([], [(k, np.zeros(n, bool)), (v, nl)])):
        out, _ = check_hash(split(cols, [0, 1000, 1500, n]), groups, [(N.AGG_FIRST_VALUE, [1])])
        assert fv.output_values(out[len(groups)]) == [1234 * 3]
    # all NULL; no keys and no rows
    out, _ = check_hash([[(k, np.zeros(n, bool)), (v, np.ones(n, bool))]], [0], [(N.AGG_FIRST_VALUE, [1])])
    assert fv.output_values(out[1]) == [None]
    a = api.HashAgg(ctx(), [N.T_INT64, N.T_FP64], [], [(N.AGG_FIRST_VALUE, [1]), (N.AGG_COUNT_STAR, [])])
    out = a.result()
    a.close()
    assert fv.output_values(out[0]) == [None] and out[1][0].tolist() == [0]
    # two groups, group 0's first row NULL: the first-row rule, not the one-group rule
    k2 = np.where(np.arange(n) == n - 1, 10, 9).astype(np.int64)
    out, _ = check_hash([[(k2, np.zeros(n, bool)), (v, nl)]], [0], [(N.AGG_FIRST_VALUE, [1])])
    assert fv.hash_output(out, 1, [1]) == {(9,): [None], (10,): [(n - 1) * 3]}


def test_hash_growth_and_overflow_rerun():
    n = 1_000_003
    cols = keys(n, 1, 400_000, 41) + values(n, 42)
    aggs = [(N.AGG_FIRST_VALUE, [1]), (N.AGG_COUNT_STAR, []), (N.AGG_FIRST_VALUE, [2])]
    _, prof = check_hash(split(cols, [0, 1, 600_000, n]), [0], aggs, expected_groups=16)
    assert "agg_rehash" in prof, prof


@pytest.mark.parametrize("nkeys", [1, 2])
def test_hash_keeps_row_order_where_the_prepass_would_run(monkeypatch, nkeys):
    """Settings that force the slot-range pre-pass on other specs: a spec with FIRST_VALUE skips it (its row tags are the
    positions as passed) and still gives every group its first row's value."""
    monkeypatch.setenv("GSQL_AGG_PARTITION_MIN_ROWS", "1000")
    monkeypatch.setenv("GSQL_AGG_PARTITION_BYTES", str(1 << 20))
    n = 1_000_003
    cols = keys(n, nkeys, 150_000, 51) + values(n, 52, nulls=0.4)
    aggs = [(N.AGG_FIRST_VALUE, [nkeys]), (N.AGG_SUM, [nkeys]), (N.AGG_FIRST_VALUE, [nkeys + 1])]
    _, prof = check_hash(split(cols, [0, 1, 300_000, n]), list(range(nkeys)), aggs, expected_groups=300_000)
    assert "agg_consume" in prof and "agg_part_scatter" not in prof, prof
    _, prof = run_hash(split(cols, [0, n]), list(range(nkeys)), [(N.AGG_SUM, [nkeys])], expected_groups=300_000)
    assert "agg_part_scatter" in prof, prof  # the same settings do reorder a spec without FIRST_VALUE


def test_filter_argument_is_refused_on_both_handles():
    t = [N.T_INT64, N.T_INT64, N.T_INT64]
    for make in (lambda **kw: api.HashAgg(ctx(), t, [0], [(N.AGG_FIRST_VALUE, [1])], **kw),
                 lambda **kw: api.SortAgg(ctx(), t, [0], [(N.AGG_FIRST_VALUE, [1])], **kw)):
        with pytest.raises(N.GsqlError) as e:
            make(filter_args=[2])
        assert e.value.status == N.E_UNSUPPORTED
    with pytest.raises(N.GsqlError) as e:
        ops.GpuHashAggExec([ops.DataTypes.LongType] * 3, [0], [ops.InternalFirstValue(1, filterArg=2)])
    assert e.value.status == N.E_UNSUPPORTED


# ------------------------------------------------------------------------------------------------ sorted aggregation
def run_sorted(cols, groups, aggs, cuts, mem="host"):
    types = [ax._type_of(d) for d, _ in cols]
    s = api.SortAgg(ctx(), types, groups, aggs)
    parts = []
    try:
        for b in split(cols, cuts):
            s.consume(to_device(b) if mem == "device" else b)
        s.finish()
        parts.append(s.next(len(cols[0][0]) + 1))
    finally:
        s.close()
    return parts[0]


def check_sorted(cols, groups, aggs, cuts, mem="host"):
    out = run_sorted(cols, groups, aggs, cuts, mem)
    vcols = [c[0] for k, c in aggs if k == N.AGG_FIRST_VALUE]
    assert fv.sorted_output(out, len(groups), fv_at(groups, aggs)) == fv.sorted_np(cols, groups, vcols)
    return out


@pytest.mark.parametrize("mem", ["host", "device"])
def test_sorted_values_bit_for_bit(mem):
    n = 40 * TILE + 13
    rng = np.random.default_rng(61)
    k = np.sort(rng.integers(0, n // 50, n)).astype(np.int64)
    cols = [(k, None)] + values(n, 62, nulls=0.7)
    aggs = [(N.AGG_FIRST_VALUE, [1]), (N.AGG_COUNT_STAR, []), (N.AGG_FIRST_VALUE, [2]), (N.AGG_FIRST_VALUE, [3])]
    check_sorted(cols, [0], aggs, [0, 1, TILE + 5, 17 * TILE, n], mem)
    check_sorted(cols, [], aggs, [0, 3 * TILE + 1, n], mem)


def test_sorted_groups_spanning_tiles_need_the_earliest_tiles_value():
    """Each long group is NULL up to a chosen row and then takes a different value in every later tile, so a continuation
    that kept a later tile's value (or the last to land) is visible.  Group lengths and NULL prefixes put the first
    non-NULL row in the head tile, in a middle tile, at a tile's first row, in a later batch, and nowhere."""
    spans = [(9 * TILE + 100, 50), (12 * TILE, 5 * TILE), (7 * TILE + 3, 3 * TILE - 7), (20 * TILE, 11 * TILE + 1),
             (6 * TILE, 6 * TILE), (3, 1), (8 * TILE + 9, 2 * TILE)]
    ks, vs, nls = [], [], []
    for g, (length, null_prefix) in enumerate(spans):
        r = np.arange(length)
        ks.append(np.full(length, g, np.int64))
        vs.append((g * 10_000_000 + r // TILE * 100 + r % 7).astype(np.int64))
        nls.append(r < null_prefix)
    cols = [(np.concatenate(ks), None), (np.concatenate(vs), np.concatenate(nls))]
    n = len(cols[0][0])
    starts = np.cumsum([0] + [s[0] for s in spans])
    # batch cuts inside the all-NULL stretch of group 3 and group 4, and just before group 6's first non-NULL row
    cuts = [0, int(starts[3] + 4 * TILE), int(starts[4] + 2 * TILE + 1), int(starts[6] + 2 * TILE - 1), n]
    out = check_sorted(cols, [0], [(N.AGG_FIRST_VALUE, [1])], cuts)
    assert fv.output_values(out[1])[4] is None
    check_sorted(cols, [0], [(N.AGG_FIRST_VALUE, [1])], [0, n], mem="device")


# ------------------------------------------------------------------------------------------------ plans
@pytest.mark.parametrize("mode", ["partial", "shuffle"])
def test_two_phase_agg_on_one_rank(mode):
    """The planner's use: values the group key determines (some NULL for the whole group), so any row order gives the
    same answer."""
    n = 300_001
    g = (ku.rand_u64(n, 71) % np.uint64(40)).astype(np.int64)
    date = g * 86_400_000 + 3                                           # DATE as a packed BIGINT
    price = np.where(g % 5 == 0, _nan(g[0] % 3 + 1), g * 0.25 - 3.0)
    nl = g % 7 == 3
    cols = [(g, np.zeros(n, bool)), (date, nl), (price, np.zeros(n, bool)), (np.ones(n, np.float64), np.zeros(n, bool))]
    calls = [(N.AGG_FIRST_VALUE, [1]), (N.AGG_FIRST_VALUE, [2]), (N.AGG_SUM, [3])]
    agg = pipelines.TwoPhaseAgg(ctx(), [N.T_INT64, N.T_INT64, N.T_FP64, N.T_FP64], [0], calls, expected_groups=64,
                                capacity=n, mode=mode, nslabs=3, nullable=[0, 1, 2, 3])
    try:
        out = to_numpy(agg.run(to_device(cols)))
    finally:
        agg.close()
    got = fv.hash_output(out, 1, [1, 2])
    assert got == fv.hash_np([cols], [0], [1, 2])
    u, cnt = np.unique(g, return_counts=True)
    assert dict(zip(np.asarray(out[0][0]).tolist(), np.asarray(out[3][0]).tolist())) == dict(zip(u.tolist(), cnt.astype(float).tolist()))


def test_operators_take_internal_first_value():
    types = [ops.DataTypes.LongType, ops.DataTypes.DoubleType]
    k = np.array([1, 1, 2, 2, 3], np.int64)
    v = np.array([0.0, -0.0, 2.5, 3.5, 0.0])
    nl = np.array([True, False, False, False, True])
    chunk = ops.Chunk(ops.LongBlock(k, None), ops.DoubleBlock(v, nl))
    h = ops.GpuHashAggExec(types, [0], [ops.InternalFirstValue(1)])
    h.consumeChunk(chunk)
    h.buildConsume()
    rows = []
    while (c := h.nextChunk()) is not None:
        rows += [tuple(r) for r in c.rows()]
    h.close()
    assert sorted(rows, key=lambda r: r[0]) == [(1, None), (2, 2.5), (3, None)]
    ex = ops.GpuSortAggExec(ops.MockExec(types, [chunk]), [0], [ops.InternalFirstValue(1)])
    rows = [tuple(r) for ch in ops.SingleExecTest(ex).exec().result() for r in ch.rows()]
    assert [r[0] for r in rows] == [1, 2, 3] and rows[1][1] == 2.5 and rows[2][1] is None
    assert struct.pack("<d", rows[0][1]) == struct.pack("<d", -0.0)  # first non-NULL, bit for bit
