"""gsql_sortagg on the GPU against the SortAggExec restatement (tests/sortagg_ref.py), row for row and in order: keys,
counts, SUM0, SUM(int) and MIN / MAX bit for bit; floating SUM / AVG exactly on dyadic data and within the gamma bound on
decimal data.  Through api.SortAgg and operators.GpuSortAggExec."""
import struct

import numpy as np
import pytest

from galaxysql_b200 import api, native as N, operators as ops
from tests import agg_exact as ax
from tests import sortagg_ref as ref
from tests.gpu_util import ctx, to_device
from tests.test_sortagg_cpu import kat_aggs, kat_chunks, kat_cols, expected_rows, ref_rows, KIND
from tests.golden.sortagg_kats import SORTAGG_KATS

pytestmark = pytest.mark.gpu

TILE = 2048  # SA_TILE of agg_sorted.cuh
ALL_INT_AGGS = lambda v: [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [v]), (N.AGG_SUM, [v]), (N.AGG_MIN, [v]), (N.AGG_MAX, [v])]


def _types(cols):
    return [ax._type_of(d) for d, _ in cols]


def run(cols, groups, aggs, splits=None, mem="host", filter_args=None, drain_every=False):
    """Consumes `cols` cut at `splits` and returns (output columns, ready counts after each consume)."""
    s = api.SortAgg(ctx(), _types(cols), groups, aggs, filter_args=filter_args)
    n = len(cols[0][0])
    cuts = [0] + list(splits or []) + [n]
    readies, parts = [], []
    try:
        for a, b in zip(cuts[:-1], cuts[1:]):
            part = [(d[a:b], None if nl is None else nl[a:b]) for d, nl in cols]
            if mem == "device":
                part = to_device(part)
            readies.append(s.consume(part))
            if drain_every and readies[-1]:
                parts.append(s.next(readies[-1]))
        readies.append(s.finish())
        parts.append(s.next(max(readies[-1], 1)))
    finally:
        s.close()
    return ref.concat(parts), readies


def check(cols, groups, aggs, mode="exact", **kw):
    want = ref.SortAggRef(cols, groups, aggs)
    got, readies = run(cols, groups, aggs, **kw)
    if want.ngroups == 0:
        assert not got
    else:
        ref.compare(got, want, mode)
    return want, readies


@pytest.mark.parametrize("case", SORTAGG_KATS, ids=lambda c: c["name"])
def test_kats_through_the_api_and_the_operator(case):
    cols = kat_cols(case)
    want = ref.SortAggRef(cols, case["groups"], kat_aggs(case), literal=True)
    got, _ = run(cols, case["groups"], kat_aggs(case), splits=[4] if len(cols[0][0]) > 4 else None)
    rows = []
    if want.ngroups:
        ref.compare(got, want)
    types = [ops.DataTypes.IntegerType if t == "int" else ops.DataTypes.DoubleType for t in case["types"]]
    chunks = [ops.Chunk(*[ops._BLOCK_OF[ops.DataTypes.IntegerType.code if t == "int" else ops.DataTypes.DoubleType.code](d, nl)
                          for (d, nl), t in zip(ch, case["types"])]) for ch in kat_chunks(case)]
    aggs = [ops.Aggregator(KIND[k], tuple(c)) for k, c in case["aggs"]]
    ex = ops.GpuSortAggExec(ops.MockExec(types, chunks), case["groups"], aggs, None, ops.ExecutionContext(chunk_size=3))
    for ch in ops.SingleExecTest(ex).exec().result():
        rows += [tuple(int(v) if isinstance(v, (int, np.integer)) else v for v in r) for r in ch.rows()]
    assert rows == expected_rows(case)


@pytest.mark.parametrize("size", [1, 2, TILE - 1, TILE, TILE + 1, 3 * TILE + 5])
def test_group_sizes_around_the_tile(size):
    n = 20 * TILE + 17
    k = (np.arange(n) // size).astype(np.int64)
    v = (ax.dyadic_numerators(n, size) % 1000).astype(np.int64)
    x, _ = ax.dyadic(ax.dyadic_numerators(n, size + 1), 4)
    cols = [(k, None), (v, ax.ku.rand_u64(n, 5) % np.uint64(7) == 0), (x, None)]
    aggs = ALL_INT_AGGS(1) + [(N.AGG_SUM0, [1]), (N.AGG_SUM, [2]), (N.AGG_AVG, [2]), (N.AGG_MIN, [2]), (N.AGG_MAX, [2])]
    check(cols, [0], aggs)
    check(cols, [0], aggs, mem="device", splits=[TILE // 2, 5 * TILE + 3])


def test_one_group_of_100m_rows():
    import torch
    n = 100_000_000
    k = torch.full((n,), 7, dtype=torch.int64, device="cuda")
    v = torch.arange(n, dtype=torch.int64, device="cuda") - n // 2
    s = api.SortAgg(ctx(), [N.T_INT64, N.T_INT64], [0], [(N.AGG_COUNT_STAR, []), (N.AGG_SUM, [1]), (N.AGG_MIN, [1]),
                                                          (N.AGG_MAX, [1]), (N.AGG_SUM0, [1])])
    assert s.consume([(k, None), (v, None)]) == 0
    out = s.result()
    s.close()
    assert out[0][0].tolist() == [7] and out[1][0].tolist() == [n]
    assert api.dec128_to_int(out[2][0]) == [sum(range(-(n // 2), n - n // 2))]
    assert out[3][0].tolist() == [-(n // 2)] and out[4][0].tolist() == [n - 1 - n // 2]
    assert out[5][0].tolist() == [ax.wrap_i64(sum(range(-(n // 2), n - n // 2)))]


def test_split_at_every_position_one_row_batches_and_empty_batches():
    rng = np.random.default_rng(3)
    n = 23
    k = np.sort(rng.integers(0, 6, n)).astype(np.int32)
    v = rng.integers(-50, 50, n).astype(np.int64)
    cols = [(k, None), (v, None)]
    aggs = ALL_INT_AGGS(1)
    want = ref.SortAggRef(cols, [0], aggs)
    for cut in range(n + 1):
        _, readies = check(cols, [0], aggs, splits=[cut])
        assert readies[0] == want.closed_before(cut)
    _, readies = check(cols, [0], aggs, splits=list(range(1, n)))
    assert readies[:-1] == [want.closed_before(r) for r in range(1, n + 1)]
    check(cols, [0], aggs, splits=[0, 0, 5, 5, 5, 12, n, n], drain_every=True)


def test_no_keys_and_no_aggregates():
    rng = np.random.default_rng(4)
    v = rng.integers(-9, 9, 10 * TILE).astype(np.int64)
    k = np.repeat(np.arange(10 * TILE // 3 + 1), 3)[:10 * TILE].astype(np.int64)
    check([(k, None), (v, None)], [], ALL_INT_AGGS(1), splits=[100, 3 * TILE])
    check([(k, None), (v, None)], [0], [], splits=[100, 3 * TILE])
    got, _ = run([(k[:0], None), (v[:0], None)], [], ALL_INT_AGGS(1))
    assert not got


def _ints(cols):
    """DEC128 columns as Python-int object arrays."""
    return [(np.array(api.dec128_to_int(d), dtype=object), nl) if np.asarray(d).ndim == 2 else (d, nl) for d, nl in cols]


def _nan(payload):
    return struct.unpack("<d", struct.pack("<q", 0x7FF8000000000000 | payload))[0]


@pytest.mark.parametrize("nkeys", [1, 2, 3, 5, 8])
def test_many_keys_with_nulls_signed_zeros_and_nan_payloads(nkeys):
    rng = np.random.default_rng(nkeys)
    n = 7 * TILE + 11
    base = np.sort(rng.integers(0, n // 3, n))
    cols = []
    for c in range(nkeys):
        t = c % 3
        if t == 0:
            d = (base // (c + 1)).astype(np.int32)
        elif t == 1:
            d = (base // (c + 1)).astype(np.int64) * 1_000_000_007
        else:
            pool = np.array([-0.0, 0.0, _nan(1), _nan(2), np.inf, -1.25], np.float64)
            d = pool[(base // (c + 1)) % 6]
            flip = rng.random(n) < 0.05  # adjacent -0.0 / +0.0 and NaN payloads inside runs
            d = np.where(flip & (d == 0), -d, d)
            d = np.where(flip & np.isnan(d), _nan(3), d)
        nl = rng.random(n) < 0.03
        cols.append((d, nl))
    x = np.where(rng.random(n) < 0.1, np.array([np.nan, -0.0, 0.0, np.inf, -np.inf])[rng.integers(0, 5, n)], rng.normal(size=n))
    cols.append((x, rng.random(n) < 0.1))
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_MIN, [nkeys]), (N.AGG_MAX, [nkeys]), (N.AGG_SUM, [nkeys]), (N.AGG_AVG, [nkeys])]
    check(cols, list(range(nkeys)), aggs, mode="bound", splits=[TILE + 1])


def test_every_aggregate_kind_with_overflow_and_avg_merge():
    n = 9 * TILE
    k = (np.arange(n) // 1000).astype(np.int64)
    big = np.where(np.arange(n) % 2 == 0, ax.INT64_MAX - np.arange(n), ax.INT64_MIN + np.arange(n)).astype(np.int64)
    big[:3000] = ax.INT64_MAX  # SUM(int) beyond +2^64, SUM0 wraps
    big[3000:6000] = ax.INT64_MIN
    ps, _ = ax.dyadic(ax.dyadic_numerators(n, 8), 3)
    pc = (np.arange(n) % 5).astype(np.int64)
    i32 = (np.arange(n) % 77 - 38).astype(np.int32)
    cols = [(k, None), (big, None), (ps, np.arange(n) % 11 == 0), (pc, np.arange(n) % 13 == 0), (i32, np.arange(n) % 3 == 0)]
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_COUNT, [1, 2]), (N.AGG_SUM, [1]), (N.AGG_SUM0, [1]), (N.AGG_MIN, [1]),
            (N.AGG_MAX, [1]), (N.AGG_AVG_MERGE, [2, 3]), (N.AGG_SUM, [4]), (N.AGG_MIN, [4]), (N.AGG_MAX, [4]),
            (N.AGG_SUM, [2]), (N.AGG_AVG, [2])]
    check(cols, [0], aggs, splits=[2999, 5 * TILE])


def test_misaligned_device_batches():
    rng = np.random.default_rng(9)
    n = 6 * TILE + 3
    k = np.sort(rng.integers(0, 300, n)).astype(np.int32)
    v = rng.integers(-5, 5, n).astype(np.int32)
    import torch
    dk = torch.from_numpy(np.r_[np.zeros(1, np.int32), k]).cuda()[1:]
    dv = torch.from_numpy(np.r_[np.zeros(1, np.int32), v]).cuda()[1:]
    s = api.SortAgg(ctx(), [N.T_INT32, N.T_INT32], [0], ALL_INT_AGGS(1))
    s.consume([(dk[:1001], None), (dv[:1001], None)])
    s.consume([(dk[1001:], None), (dv[1001:], None)])
    got = s.result()
    s.close()
    ref.compare(got, ref.SortAggRef([(k, None), (v, None)], [0], ALL_INT_AGGS(1)))


def test_next_interleaved_with_consume_returns_groups_in_order():
    n = 5 * TILE
    k = (np.arange(n) // 37).astype(np.int64)
    cols = [(k, None), ((np.arange(n) % 9).astype(np.int64), None)]
    aggs = ALL_INT_AGGS(1)
    want = ref.SortAggRef(cols, [0], aggs)
    s = api.SortAgg(ctx(), [N.T_INT64, N.T_INT64], [0], aggs)
    parts, taken = [], 0
    for a, b in [(0, 100), (100, 3000), (3000, 3001), (3001, n)]:
        ready = s.consume([(cols[0][0][a:b], None), (cols[1][0][a:b], None)])
        assert ready == want.closed_before(b) - taken
        if ready > 1:
            parts.append(s.next(ready // 2))  # part of what is ready; the rest stays for later
            taken += len(parts[-1][0][0])
    s.finish()
    parts.append(s.next(n))
    s.close()
    ref.compare(ref.concat(parts), want)


def test_errors():
    c = ctx()
    t = [N.T_INT64, N.T_INT64]
    for kw in (dict(filter_args=[1]), dict(derived=[(N.EXPR_MUL_1MINUS, 0, 1, 0)]), dict(row_filter=(1, N.CMP_GT, 3))):
        with pytest.raises(N.GsqlError) as e:
            api.SortAgg(c, t, [0], [(N.AGG_SUM, [1])], **kw)
        assert e.value.status == N.E_UNSUPPORTED
    with pytest.raises(N.GsqlError) as e:
        api.SortAgg(c, [N.T_INT64, N.T_DEC128], [0], [(N.AGG_COUNT_STAR, [])])
    assert e.value.status == N.E_UNSUPPORTED
    s = api.SortAgg(c, t, [0], [(N.AGG_SUM, [1])])
    k = np.array([1, 1, 2], np.int64)
    s.consume([(k, None), (np.array([5, 6, 7], np.int64), np.array([0, 0, 1], bool))])
    s.finish()
    with pytest.raises(N.GsqlError) as e:
        s.consume([(k, None), (k, None)])
    assert e.value.status == N.E_STATE
    with pytest.raises(N.GsqlError) as e:  # the second group's SUM is NULL: an out column without nulls cannot take it
        s.next(5, nullable_out=False)
    assert e.value.status == N.E_INVALID
    got = s.next(5)  # the cursor did not move
    s.close()
    assert got[0][0].tolist() == [1, 2] and api.dec128_to_int(got[1][0]) == [11, 0] and got[1][1].tolist() == [0, 1]


def test_after_merge_and_after_sort_equals_the_hash_agg():
    rng = np.random.default_rng(11)
    runs = []
    for _ in range(4):
        m = 3 * TILE + int(rng.integers(0, 999))
        runs.append([(np.sort(rng.integers(0, 2000, m)).astype(np.int64), None),
                     (rng.integers(-1000, 1000, m).astype(np.int64), None)])
    aggs = ALL_INT_AGGS(1)
    types = [N.T_INT64, N.T_INT64]
    mg = api.Merge(ctx(), types, [0], [False], len(runs))
    for i, r in enumerate(runs):
        mg.consume(i, r)
    merged = mg.result()
    mg.close()
    allrows = [(np.concatenate([r[c][0] for r in runs]), None) for c in range(2)]
    perm = np.random.default_rng(1).permutation(len(allrows[0][0]))
    so = api.Sort(ctx(), types, [0], [True])
    so.consume([(allrows[0][0][perm], None), (allrows[1][0][perm], None)])
    sorted_ = so.result()
    so.close()
    h = api.HashAgg(ctx(), types, [0], aggs)
    h.consume(allrows)
    hash_rows = ax.result_by_key(_ints(h.result()), 1)
    h.close()
    for src in (merged, sorted_):
        src = [(np.asarray(d), None if nl is None else np.asarray(nl)) for d, nl in src]
        got, _ = run(src, [0], aggs, splits=[TILE + 7])
        ref.compare(got, ref.SortAggRef(src, [0], aggs))
        assert ax.result_by_key(_ints(got), 1) == hash_rows


def test_profile_shows_the_tile_kernel():
    c = ctx()
    c.profile(True)
    c.profile_reset()
    check([(np.arange(3 * TILE, dtype=np.int64) // 5, None), (np.ones(3 * TILE, np.int64), None)], [0], ALL_INT_AGGS(1))
    prof = c.profile_dump()
    c.profile(False)
    assert prof.get("sagg_tile", (0, 0))[0] >= 1 and prof.get("sagg_fixup", (0, 0))[0] >= 1
