"""-m gpu checks of ORDER BY / TOP-N (gsql_sort_*, api.Sort, operators.GpuSortExec / GpuTopNExec) against the two
restatements of the executor's comparator in tests/sort_ref.py.  Every output is checked the same way
(sort_ref.check_ordered): the key sequence is the reference's exactly, the rows are a sub-multiset of the input (the
input itself for a full sort), and every row strictly ahead of the last key kept is present.  Cases also assert from
the kernel profile that the intended path ran."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

from galaxysql_b200 import api, native as N
from tests import sort_ref as sr
from tests.golden import sort_kats

pytestmark = pytest.mark.gpu

F64_SPECIALS = np.array([0x8000000000000000, 0, 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000001,
                         0xFFFFFFFFFFFFFFFF, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF,
                         0x0000000000000001, 0x8000000000000001, 0x000FFFFFFFFFFFFF, 0x3FF0000000000000],
                        dtype=np.uint64).view(np.float64)
I64_SPECIALS = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).min + 1, -1, 0, 1, np.iinfo(np.int64).max - 1,
                         np.iinfo(np.int64).max, np.iinfo(np.int32).min, np.iinfo(np.int32).max], dtype=np.int64)
I32_SPECIALS = np.array([np.iinfo(np.int32).min, np.iinfo(np.int32).min + 1, -1, 0, 1, np.iinfo(np.int32).max], dtype=np.int32)


@pytest.fixture(scope="module")
def ctx():
    from tests import gpu_util
    return gpu_util.ctx()


def _types(cols):
    m = {np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}
    return [m[np.asarray(d).dtype] for d, _ in cols]


def _dev(cols):
    from tests import gpu_util
    return gpu_util.to_device(cols)


def _np(cols):
    from tests import gpu_util
    return gpu_util.to_numpy(cols)


def run(ctx, cols, keys, desc, limit=None, parts=1, mem="host", out_mem=N.MEM_HOST, chunk=None):
    """Consumes `cols` in `parts` batches (mem: host / device / mixed) and returns the ordered rows as numpy columns."""
    types = _types(cols)
    s = api.Sort(ctx, types, keys, desc, limit)
    n = len(cols[0][0])
    bounds = np.linspace(0, n, parts + 1).astype(int)
    for p in range(parts):
        piece = [(d[bounds[p]:bounds[p + 1]], None if nl is None else nl[bounds[p]:bounds[p + 1]]) for d, nl in cols]
        m = mem if mem != "mixed" else ("device" if p % 2 else "host")
        s.consume(_dev(piece) if m == "device" else piece)
    total = s.finish()
    outs = []
    while True:
        o = s.next(chunk or max(total, 1), out_mem)
        if len(o[0][0]) == 0:
            break
        outs.append(_np(o))
    s.close()
    if not outs:
        return [(np.zeros(0, np.asarray(d).dtype), np.zeros(0, bool)) for d, _ in cols]
    return [(np.concatenate([o[c][0] for o in outs]), np.concatenate([o[c][1] for o in outs])) for c in range(len(cols))]


def check(ctx, cols, keys, desc, limit=None, **kw):
    """Runs the sort under the kernel profile, checks the output, and asserts that the intended path ran: nothing for an
    empty input or LIMIT 0, the radix select for a LIMIT below the row count, otherwise the full sort (whose digit passes
    are skipped only when every key is constant).  The profile is left in check.prof."""
    ctx.profile(True)
    ctx.profile_reset()
    try:
        out = run(ctx, cols, keys, desc, limit, **kw)
        prof = ctx.profile_dump()
    finally:
        ctx.profile(False)
    sr.check_ordered(out, cols, _types(cols), keys, desc, limit)
    n = len(cols[0][0])
    km = sr.key_matrix(cols, _types(cols), keys)
    constant = n <= 1 or bool((km == km[0]).all())
    if n == 0 or limit == 0:
        assert not any(k.startswith(("k_sort", "k_topn")) for k in prof), prof
    else:
        assert "k_sort_minmax" in prof and "k_sort_gather" in prof, prof
        if limit is not None and limit < n and not constant:
            assert all(k in prof for k in ("k_topn_hist", "k_topn_pick", "k_topn_compact")), prof
        else:
            assert "k_topn_hist" not in prof, prof
            assert ("k_sort_radix" in prof) == (not constant), prof
    check.prof = prof
    return out


def profiled(ctx, fn):
    ctx.profile(True)
    ctx.profile_reset()
    fn()
    prof = ctx.profile_dump()
    ctx.profile(False)
    return prof


def _rand(n, seed, dtype, lo=None, hi=None, null_frac=0.0):
    rng = np.random.default_rng(seed)
    if dtype == np.float64:
        v = rng.standard_normal(n) * 1e6
    else:
        info = np.iinfo(dtype)
        v = rng.integers(info.min if lo is None else lo, (info.max if hi is None else hi), n, dtype=dtype, endpoint=True)
    nl = rng.random(n) < null_frac if null_frac else None
    return v, nl


# ------------------------------------------------------------------------------------------------ key order
@pytest.mark.parametrize("specials", [F64_SPECIALS, I64_SPECIALS, I32_SPECIALS], ids=["fp64", "int64", "int32"])
@pytest.mark.parametrize("desc", [False, True])
def test_every_ordered_pair_of_special_values(ctx, specials, desc):
    vals = list(specials) + [None]
    for a in vals:
        for b in vals:
            v = np.array([0 if x is None else x for x in (a, b)], dtype=specials.dtype)
            nl = np.array([a is None, b is None])
            check(ctx, [(v, nl if nl.any() else None), (np.arange(2, dtype=np.int32), None)], [0], [desc])
    # and all of them at once, repeated, with a second key breaking ties
    v = np.tile(specials, 7)
    nl = np.arange(len(v)) % 5 == 0
    check(ctx, [(v, nl), (np.arange(len(v), dtype=np.int64) % 3, None)], [0, 1], [desc, not desc])


@pytest.mark.parametrize("desc", [False, True])
def test_nulls_lead_under_asc_and_trail_under_desc(ctx, desc):
    v, nl = _rand(100_000, 3, np.int64, -50, 50, null_frac=0.1)
    out = check(ctx, [(v, nl), (np.arange(len(v), dtype=np.int32), None)], [0], [desc])
    k = int(nl.sum())
    assert out[0][1][:k].all() != desc and out[0][1][len(v) - k:].all() == desc


@pytest.mark.parametrize("nkeys", range(1, 9))
def test_one_to_eight_keys_with_mixed_directions(ctx, nkeys):
    rng = np.random.default_rng(nkeys)
    n = 200_000
    cols = []
    for c in range(8):
        dt = [np.int32, np.int64, np.float64][c % 3]
        if dt == np.float64:
            v = rng.choice(F64_SPECIALS, n) if c % 2 else np.round(rng.standard_normal(n), 1)
        else:  # few distinct values so that later keys decide
            v = rng.choice(I64_SPECIALS if dt == np.int64 else I32_SPECIALS, n).astype(dt) if c % 2 else rng.integers(-3, 3, n).astype(dt)
        cols.append((v, rng.random(n) < 0.05 if c % 3 == 1 else None))
    keys = list(rng.permutation(8)[:nkeys])
    desc = list(rng.random(nkeys) < 0.5)
    check(ctx, cols, keys, desc)


def test_groups_beyond_128_bits(ctx):
    """8 full-range BIGINT keys: 512 bits, at least 4 images of <= 128 bits, sorted least significant first."""
    rng = np.random.default_rng(11)
    n = 100_000
    base = rng.integers(0, 4, (n, 8))  # a few values per key so that every key matters...
    spread = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, 8, dtype=np.int64, endpoint=True)
    cols = [(np.where(base[:, c] == 3, spread[c], base[:, c] - (np.int64(1) << 62)).astype(np.int64), None) for c in range(8)]
    for c in range(8):  # ...and full-width ranges: min and max of int64 present in each key
        cols[c][0][c] = np.iinfo(np.int64).min
        cols[c][0][c + 8] = np.iinfo(np.int64).max
    desc = [bool(c % 2) for c in range(8)]
    check(ctx, cols, list(range(8)), desc)
    prof = check.prof
    assert prof["k_sort_radix"][0] >= 4 and prof["k_sort_encode"][0] == prof["k_sort_radix"][0]


@pytest.mark.parametrize("k", [1, 7, 12, 31, 32, 33, 63])
def test_integer_ranges_at_power_of_two_boundaries(ctx, k):
    rng = np.random.default_rng(k)
    for span in ((1 << k) - 1, 1 << k):
        lo = -(1 << 62) if k < 62 else -(1 << 63)
        off = rng.integers(0, span, 50_000, dtype=np.uint64, endpoint=True)
        v = (np.uint64(lo % (1 << 64)) + off).view(np.int64)
        v[0], v[1] = lo, lo + span
        check(ctx, [(v, None)], [0], [False])
        check(ctx, [(v, None)], [0], [True], limit=100)


def test_full_64_bit_range_and_a_single_value(ctx):
    v = np.concatenate([I64_SPECIALS, _rand(10_000, 5, np.int64)[0]])
    check(ctx, [(v, None)], [0], [False])
    one = np.full(5000, 42, np.int64)
    check(ctx, [(one, None), (np.arange(5000, dtype=np.int32), None)], [0], [True])
    prof = check.prof
    assert "k_sort_radix" not in prof  # a constant key needs no digit pass


# ------------------------------------------------------------------------------------------------ batch shapes
@pytest.mark.parametrize("n", [0, 1])
@pytest.mark.parametrize("limit", [None, 0, 1, 5])
def test_zero_and_one_row(ctx, n, limit):
    cols = [(np.arange(n, dtype=np.int64), None), (np.ones(n), None)]
    check(ctx, cols, [0], [True], limit)


@pytest.mark.parametrize("limit", [None, 10, 5000])
def test_many_batches_mixing_host_and_device(ctx, limit):
    v, nl = _rand(300_000, 9, np.float64, null_frac=0.02)
    i, _ = _rand(300_000, 10, np.int32, -5, 5)
    for mem in ("host", "device", "mixed"):
        check(ctx, [(v, nl), (i, None)], [1, 0], [False, True], limit, parts=7, mem=mem)
    check(ctx, [(v, nl), (i, None)], [1, 0], [False, True], limit, parts=3, mem="mixed", out_mem=N.MEM_DEVICE, chunk=777)


def test_misaligned_device_views(ctx):
    import torch
    v, nl = _rand(10_001, 12, np.int64, -1000, 1000, null_frac=0.1)
    w, _ = _rand(10_001, 13, np.int32)
    dv, dn, dw = torch.from_numpy(v).cuda(), torch.from_numpy(nl.astype(np.uint8)).cuda(), torch.from_numpy(w).cuda()
    for off in (1, 3):
        s = api.Sort(ctx, [N.T_INT64, N.T_INT32], [0, 1], [True, False])
        s.consume([(dv[off:], dn[off:]), (dw[off:], None)])
        out = _np(s.result(N.MEM_DEVICE))
        s.close()
        sr.check_ordered(out, [(v[off:], nl[off:]), (w[off:], None)], [N.T_INT64, N.T_INT32], [0, 1], [True, False])


# ------------------------------------------------------------------------------------------------ top-n
@pytest.mark.parametrize("limit_of", [lambda r: 0, lambda r: 1, lambda r: r, lambda r: r + 5], ids=["0", "1", "R", "gtR"])
def test_topn_limits(ctx, limit_of):
    v, nl = _rand(123_457, 14, np.float64, null_frac=0.01)
    check(ctx, [(v, nl), (np.arange(len(v), dtype=np.int64), None)], [0], [True], limit_of(len(v)))


def test_topn_ties_at_the_boundary(ctx):
    v = np.repeat(np.arange(1000, dtype=np.int32), 100)  # every key 100 times
    np.random.default_rng(1).shuffle(v)
    for limit in (1, 150, 4321, 50_050):
        check(ctx, [(v, None), (np.arange(len(v), dtype=np.int64), None)], [0], [False], limit)


@pytest.mark.parametrize("odd", [None, "min", "max"])
def test_topn_refines_equal_leading_keys(ctx, odd):
    """All-equal (or all-but-one-equal) leading keys: the first histogram level cannot cut, so the selection refines."""
    n = 1 << 20
    lead = np.full(n, 7, np.int64)
    if odd == "min":
        lead[n // 3] = -7
    elif odd == "max":
        lead[n // 3] = 1 << 40
    second = np.random.default_rng(2).integers(0, 1 << 30, n).astype(np.int64)
    check(ctx, [(lead, None), (second, None)], [0, 1], [False, False], 100)
    prof = check.prof
    # a constant leading key drops out of the image and the second key is selected on; otherwise the first 11-bit digit
    # keeps (almost) every row and later levels cut
    assert prof["k_topn_hist"][0] >= 2 and prof["k_topn_compact"][0] == prof["k_topn_hist"][0]


def test_topn_50m_rows(ctx):
    import torch
    n = 50_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    v = torch.randn(n, device="cuda", dtype=torch.float64, generator=g)
    s = api.Sort(ctx, [N.T_FP64], [0], [True], 1000)

    def go():
        s.consume([(v, None)])
        return s.result()
    prof = profiled(ctx, lambda: setattr(s, "_out", go()))
    out = s._out
    s.close()
    ref = torch.topk(v, 1000).values.cpu().numpy()
    assert np.array_equal(out[0][0], ref)
    assert prof["k_topn_hist"][0] >= 1 and prof["k_topn_compact"][0] >= 1 and prof["k_topn_pick"][0] >= 1


def test_topn_holds_o_of_limit_rows_across_batches(ctx):
    v, nl = _rand(2_000_000, 15, np.int64, null_frac=0.01)
    check(ctx, [(v, nl)], [0], [True], 1000, parts=40, mem="mixed")


# ------------------------------------------------------------------------------------------------ errors
def test_argument_errors(ctx):
    with pytest.raises(N.GsqlError) as e:
        api.Sort(ctx, [N.T_INT64, N.T_DEC128], [0], [False])
    assert e.value.status == N.E_UNSUPPORTED and "DEC128" in str(e.value)
    for bad in (dict(keys=[2]), dict(keys=[]), dict(limit=-2)):
        with pytest.raises(N.GsqlError) as e:
            api.Sort(ctx, [N.T_INT64, N.T_FP64], bad.get("keys", [0]), [False] * len(bad.get("keys", [0])), bad.get("limit"))
        assert e.value.status == N.E_INVALID
    s = api.Sort(ctx, [N.T_INT64], [0], [False])
    s.consume([(np.array([3, 1, 2], np.int64), np.array([0, 1, 0], bool))])
    assert s.finish() == 3
    with pytest.raises(N.GsqlError) as e:
        s.next(3, N.MEM_HOST, nullable_out=False)
    assert e.value.status == N.E_INVALID
    out = s.next(3)  # the cursor did not move
    assert out[0][1].tolist() == [1, 0, 0] and out[0][0][1:].tolist() == [2, 3]
    with pytest.raises(N.GsqlError) as e:
        s.consume([(np.array([1], np.int64), None)])
    assert e.value.status == N.E_STATE
    s.close()


# ------------------------------------------------------------------------------------------------ reference KATs
@pytest.mark.parametrize("kat", sort_kats.ALL_KATS, ids=lambda k: k["name"])
def test_reference_kats_through_the_operators(ctx, kat):
    from galaxysql_b200 import operators as ops
    T = ops.DataTypes.IntegerType
    chunks = [ops.Chunk(*[ops.IntegerBlock.of(*col) for col in ch]) for ch in kat["chunks"]]
    src = ops.MockExec.builder(T, T)
    for ch in chunks:
        src.withChunk(ch)
    src = src.build()
    orders = [ops.OrderByOption(c, ops.Direction.DESCENDING if d else ops.Direction.ASCENDING, nd) for c, d, nd in kat["order"]]
    ectx = ops.ExecutionContext(chunk_size=3)
    exec_ = ops.GpuSortExec(src.getDataTypes(), orders, ectx) if kat["top"] is None else ops.GpuTopNExec(src.getDataTypes(), orders, kat["top"], ectx)
    rows = [r for ch in ops.SingleExecTest(exec_, src).exec().result() for r in ch.rows()]
    exp = list(zip(*kat["expect"]))
    if kat["ordered"]:
        assert rows == exp
    else:
        assert Counter(rows) == Counter(exp)
