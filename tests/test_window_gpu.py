"""gsql_window on the GPU against the NonFrameOverWindowExec restatement (tests/window_ref.py), row for row and in order:
the rank family, counts, SUM0, SUM(int) and MIN / MAX bit for bit; floating SUM / AVG exactly on dyadic data and within
the gamma bound on decimal data.  Through api.Window and operators.GpuNonFrameOverWindowExec."""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest

from galaxysql_b200 import api, native as N, operators as ops
from tests.golden import window_kats as K
from tests.gpu_util import ctx, to_device
from tests.window_ref import window_np, window_rows

pytestmark = pytest.mark.gpu

TILE = 1024  # WT_TILE of window.cuh
KIND = {"ROW_NUMBER": N.AGG_ROW_NUMBER, "RANK": N.AGG_RANK, "DENSE_RANK": N.AGG_DENSE_RANK, "COUNT_STAR": N.AGG_COUNT_STAR,
        "COUNT": N.AGG_COUNT, "SUM": N.AGG_SUM, "SUM0": N.AGG_SUM0, "AVG": N.AGG_AVG, "MIN": N.AGG_MIN, "MAX": N.AGG_MAX}
_T = {np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def run(cols, part, calls, splits=None, mem="host", out_mem=None, reset=False):
    """Applies the window to `cols` cut at `splits` -> one Python list per call (None = NULL)."""
    w = api.Window(ctx(), [_T[d.dtype] for d, _ in cols], part, [(KIND[k], c) for k, c in calls], reset_each_row=reset)
    n = len(cols[0][0])
    cuts = [0] + list(splits or []) + [n]
    got = [[] for _ in calls]
    try:
        for a, b in zip(cuts[:-1], cuts[1:]):
            piece = [(d[a:b], None if nl is None else nl[a:b]) for d, nl in cols]
            if mem == "device":
                piece = to_device(piece)
            res = w.apply(piece, mem=out_mem)
            for i, ((d, nl), t) in enumerate(zip(res, w.out_types)):
                d = d.cpu().numpy() if hasattr(d, "cpu") else d
                nl = nl.cpu().numpy() if hasattr(nl, "cpu") else nl
                vals = api.dec128_to_int(d) if t == N.T_DEC128 else d.tolist()
                got[i].extend(None if nl[r] else vals[r] for r in range(len(vals)))
    finally:
        w.close()
    return got


def expected(cols, part, calls, splits=None, reset=False):
    n = len(cols[0][0])
    cuts = [0] + list(splits or []) + [n]
    batches = [[(d[a:b], None if nl is None else nl[a:b]) for d, nl in cols] for a, b in zip(cuts[:-1], cuts[1:])]
    exp = window_rows(batches, part, calls, reset)
    for i, (k, c) in enumerate(calls):  # documented divergence: an all -0.0 DOUBLE sum is +0.0 on the GPU
        if k in ("SUM", "AVG") and c and cols[c[0]][0].dtype == np.float64:
            exp[i] = [0.0 if (v == 0.0 and math.copysign(1, v) < 0) else v for v in exp[i]]
    return exp


def same(got, exp):
    """Bit for bit, NaN payloads aside (MIN / MAX return the canonical NaN, as gsql_agg does)."""
    assert len(got) == len(exp)
    for g, e in zip(got, exp):
        assert len(g) == len(e)
        for r, (a, b) in enumerate(zip(g, e)):
            if isinstance(b, float):
                assert a is not None and (_bits(a) == _bits(b) or (math.isnan(a) and math.isnan(b))), (r, a, b)
            else:
                assert a == b, (r, a, b)


def check(cols, part, calls, **kw):
    same(run(cols, part, calls, **kw), expected(cols, part, calls, kw.get("splits"), kw.get("reset", False)))


def _runs(lengths, rng):
    p = np.repeat(np.arange(len(lengths), dtype=np.int64), lengths)
    o = np.concatenate([np.sort(rng.integers(0, max(2, n // 3), n)) for n in lengths]).astype(np.int64)
    return p, o


INT_CALLS = [("ROW_NUMBER", []), ("RANK", [1]), ("DENSE_RANK", [1]), ("COUNT_STAR", []), ("COUNT", [2]), ("SUM", [2]),
             ("SUM0", [2]), ("MIN", [2]), ("MAX", [2])]


@pytest.mark.parametrize("case", K.CASES, ids=[c[0] for c in K.CASES])
def test_reference_kats(case):
    name, part, calls, reset, exp = case
    rows = [r for ch in K.NORMAL for r in ch]
    splits = list(np.cumsum([len(ch) for ch in K.NORMAL])[:-1])
    dt = [np.float64 if name == "testAvgV2AndCountV2" else np.int64] * 3
    cols = [(np.array([0 if r[c] is None else r[c] for r in rows], dt[c]), np.array([r[c] is None for r in rows], np.uint8))
            for c in range(3)]
    for i, (call, e) in enumerate(zip(calls, exp)):  # one flag per operator: the calls run one by one
        got = run(cols, part, [call], splits=splits, reset=reset[i])[0]
        assert got == [float(x) if isinstance(x, Fraction) else x for x in e]


@pytest.mark.parametrize("size", [1, TILE - 1, TILE, TILE + 1])
def test_partition_sizes_around_the_tile(size):
    rng = np.random.default_rng(size)
    p, o = _runs([size] * (5 * TILE // size + 3), rng)
    v = rng.integers(-1000, 1000, len(p)).astype(np.int64)
    nl = (rng.random(len(p)) < 0.1).astype(np.uint8)
    check([(p, None), (o, None), (v, nl)], [0], INT_CALLS)


def test_one_partition_of_100m_rows():
    n = 100_000_000
    rng = np.random.default_rng(3)
    p = np.zeros(n, np.int64)
    o = np.repeat(np.arange(n // 7 + 1, dtype=np.int64), 7)[:n]
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    cols = [(p, None), (o, None), (v, None)]
    calls = [("ROW_NUMBER", []), ("RANK", [1]), ("DENSE_RANK", [1])]
    w = api.Window(ctx(), [N.T_INT64] * 3, [0], [(KIND[k], c) for k, c in calls] + [(N.AGG_SUM0, [2])])
    try:
        res = w.apply(to_device(cols))
        exp = window_np(cols, [0], calls + [("SUM", [2])])
        for (d, nl), e in zip(res, exp):
            d = d.cpu().numpy()
            assert not nl.cpu().numpy().any()
            assert np.array_equal(d, e)
    finally:
        w.close()


def test_splits_at_every_position_one_row_and_empty_batches():
    rng = np.random.default_rng(11)
    n = 40
    p, o = _runs([3, 1, 7, 2, 9, 1, 5, 12], rng)
    v = rng.integers(-9, 9, n).astype(np.int64)
    nl = (rng.random(n) < 0.2).astype(np.uint8)
    cols = [(p, nl.copy()), (o, None), (v, nl)]
    for s in range(n + 1):
        check(cols, [0], INT_CALLS, splits=[s])
    check(cols, [0], INT_CALLS, splits=list(range(1, n)))
    check(cols, [0], INT_CALLS, splits=[0, 0, 5, 5, n, n], mem="device")


def test_null_zero_and_nan_payload_keys():
    nan2 = struct.unpack("<d", struct.pack("<q", 0x7ff8000000000abc))[0]
    vals = [0.0, -0.0, math.nan, nan2, 1.5, None]
    rng = np.random.default_rng(5)
    n = 5 * TILE + 17
    pick = rng.integers(0, len(vals), n)
    pick.sort()
    keys = np.array([0.0 if vals[i] is None else vals[i] for i in pick], np.float64)
    knull = np.array([vals[i] is None for i in pick], np.uint8)
    opick = rng.integers(0, len(vals), n)
    okeys = np.array([0.0 if vals[i] is None else vals[i] for i in opick], np.float64)
    onull = np.array([vals[i] is None for i in opick], np.uint8)
    x = rng.integers(0, 100, n).astype(np.int32)
    cols = [(keys, knull), (okeys, onull), (x, None)]
    calls = [("ROW_NUMBER", []), ("RANK", [1, 2]), ("DENSE_RANK", [1]), ("SUM", [2]), ("MIN", [1]), ("MAX", [1])]
    check(cols, [0], calls, splits=[TILE + 3, 3 * TILE])
    check(cols, [0, 2], calls, mem="device")


def test_every_kind_and_sum_crossing_2_pow_64():
    rng = np.random.default_rng(9)
    n = 3 * TILE + 5
    p = np.sort(rng.integers(0, 4, n)).astype(np.int32)
    big = np.where(rng.random(n) < 0.5, np.iinfo(np.int64).max - rng.integers(0, 5, n), np.iinfo(np.int64).min + rng.integers(0, 5, n))
    big[: 2 * TILE] = np.iinfo(np.int64).max
    nl = (rng.random(n) < 0.05).astype(np.uint8)
    d = (rng.integers(-2 ** 20, 2 ** 20, n) / 256.0).astype(np.float64)
    i32 = rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32)
    cols = [(p, None), (big.astype(np.int64), nl), (d, nl), (i32, None)]
    calls = [("ROW_NUMBER", []), ("RANK", [3]), ("DENSE_RANK", [3]), ("COUNT_STAR", []), ("COUNT", [1, 2]),
             ("SUM", [1]), ("SUM", [3]), ("SUM0", [1]), ("SUM", [2]), ("AVG", [2]), ("MIN", [2]), ("MAX", [2]),
             ("MIN", [3]), ("MAX", [1])]
    check(cols, [0], calls, splits=[TILE // 2, 2 * TILE + 1])
    check(cols, [0], calls, reset=True)
    check(cols, [], calls, mem="device", out_mem=N.MEM_HOST)


def test_dyadic_sums_exact_and_decimal_sums_within_gamma():
    rng = np.random.default_rng(21)
    n = 20_000
    p = np.repeat(np.arange(4, dtype=np.int64), n // 4)
    dy = rng.integers(-2 ** 30, 2 ** 30, n) * 2.0 ** -20
    check([(p, None), (dy, None)], [0], [("SUM", [1]), ("AVG", [1])], splits=[3333])
    dec = np.round(rng.uniform(-1e6, 1e6, n), 2)
    cols = [(p, None), (dec, None)]
    got = run(cols, [0], [("SUM", [1]), ("AVG", [1])], splits=[7777])
    exact = window_rows([cols], [0], [("SUM", [1])], exact=True)[0]
    absum = window_rows([[(p, None), (np.abs(dec), None)]], [0], [("SUM", [1]), ("COUNT_STAR", [])], exact=True)
    u = 2.0 ** -53
    for r in range(n):
        k = absum[1][r]
        g = (k - 1) * u / (1 - (k - 1) * u)
        assert abs(Fraction(got[0][r]) - exact[r]) <= g * absum[0][r]
        assert abs(Fraction(got[1][r]) - exact[r] / k) <= (g + 2 * u) * absum[0][r] / k


def test_misaligned_device_batches_and_host_device_mixes():
    import torch
    rng = np.random.default_rng(13)
    n = 4 * TILE + 9
    p, o = _runs([n // 5] * 5 + [n - 5 * (n // 5)], rng)
    v = rng.integers(-50, 50, n).astype(np.int64)
    cols = [(p, None), (o, None), (v, None)]
    exp = expected(cols, [0], INT_CALLS)
    dev = to_device(cols)
    shifted = []
    for d, _ in dev:  # one element past a 256-byte-aligned allocation
        big = torch.empty(len(d) + 1, dtype=d.dtype, device=d.device)
        big[1:] = d
        shifted.append((big[1:], None))
    w = api.Window(ctx(), [N.T_INT64] * 3, [0], [(KIND[k], c) for k, c in INT_CALLS])
    try:
        got = [[] for _ in INT_CALLS]
        for a, b in [(0, 1001), (1001, n)]:
            res = w.apply([(d[a:b], None) for d, _ in shifted], mem=N.MEM_DEVICE if a == 0 else N.MEM_HOST)
            for i, (d, nl) in enumerate(res):
                d = d.cpu().numpy() if hasattr(d, "cpu") else d
                nl = nl.cpu().numpy() if hasattr(nl, "cpu") else nl
                vals = api.dec128_to_int(d) if w.out_types[i] == N.T_DEC128 else d.tolist()
                got[i].extend(None if nl[r] else vals[r] for r in range(len(vals)))
    finally:
        w.close()
    same(got, exp)
    check(cols, [0], INT_CALLS, splits=[777], mem="host", out_mem=N.MEM_DEVICE)


@pytest.mark.parametrize("offset", [1, 3, 4, 7])
def test_device_bases_not_aligned_to_their_element(offset):
    """Columns placed `offset` bytes into a device buffer: 8-byte columns then go through the byte-copy staging (and the
    carry's byte loads); 4-byte ones too unless offset is 4.  A misaligned output column is refused."""
    import ctypes as C
    import torch
    rng = np.random.default_rng(offset)
    n = 3 * TILE + 77
    p, o = _runs([5, TILE + 3, 1, 700, n - TILE - 709], rng)
    onl = (rng.random(n) < 0.1).astype(np.uint8)
    o = np.where(onl == 1, 0, o)
    v = rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32)
    d = (rng.integers(-2 ** 20, 2 ** 20, n) / 64.0).astype(np.float64)
    cols = [(p, None), (o, onl), (v, None), (d, None)]
    calls = [("ROW_NUMBER", []), ("RANK", [1]), ("DENSE_RANK", [1]), ("SUM", [2]), ("SUM", [3]), ("MIN", [3]), ("MAX", [2])]
    splits = [TILE + 5, 2 * TILE]
    exp = expected(cols, [0], calls, splits)
    c = ctx()
    keep = []

    def place(arr):
        b = np.ascontiguousarray(arr).view(np.uint8)
        buf = torch.zeros(len(b) + 16, dtype=torch.uint8, device=f"cuda:{c.device}")
        buf[offset:offset + len(b)] = torch.from_numpy(b.copy()).to(buf.device)
        keep.append(buf)
        return buf.data_ptr() + offset

    w = api.Window(c, [N.T_INT64, N.T_INT64, N.T_INT32, N.T_FP64], [0], [(KIND[k], cc) for k, cc in calls])
    got = [[] for _ in calls]
    try:
        for a, b in zip([0] + splits, splits + [n]):
            carr = (N.Col * len(cols))()
            for i, (data, nl) in enumerate(cols):
                carr[i].type = _T[data.dtype]
                carr[i].data = place(data[a:b])
                carr[i].nulls = 0 if nl is None else place(nl[a:b])
            torch.cuda.synchronize()
            batch = N.Batch(b - a, len(cols), N.MEM_DEVICE, carr)
            out = api._alloc_out(c, w.out_types, b - a, N.MEM_DEVICE, [True] * len(calls))
            ob, _k = api._out_batch(out, w.out_types, 0, N.MEM_DEVICE)
            c.check(c.lib.gsql_window_apply(w.h, C.byref(batch), C.byref(ob)))
            c.sync()
            for i, ((dd, nn), t) in enumerate(zip(api._trim(out, b - a), w.out_types)):
                dd, nn = dd.cpu().numpy(), nn.cpu().numpy()
                vals = api.dec128_to_int(dd) if t == N.T_DEC128 else dd.tolist()
                got[i].extend(None if nn[r] else vals[r] for r in range(len(vals)))
        same(got, exp)
        out = api._alloc_out(c, w.out_types, 8, N.MEM_DEVICE, [True] * len(calls))
        ob, _k = api._out_batch(out, w.out_types, 0, N.MEM_DEVICE)
        ob.cols[0].data += 4  # ROW_NUMBER's BIGINT column, 4 bytes off its element
        batch = N.Batch(0, len(cols), N.MEM_DEVICE, carr)
        assert c.lib.gsql_window_apply(w.h, C.byref(batch), C.byref(ob)) == N.E_INVALID
    finally:
        w.close()


def test_sort_then_window():
    rng = np.random.default_rng(17)
    n = 6 * TILE + 11
    p = rng.integers(0, 50, n).astype(np.int64)
    o = rng.integers(0, 20, n).astype(np.int64)
    v = rng.integers(-100, 100, n).astype(np.int64)
    s = api.Sort(ctx(), [N.T_INT64] * 3, [0, 1])
    s.consume([(p, None), (o, None), (v, None)])
    sorted_cols = s.result()
    s.close()
    cols = [(np.asarray(d), None) for d, _ in sorted_cols]
    assert np.all(np.diff(cols[0][0]) >= 0)
    check(cols, [0], INT_CALLS, mem="device")


@pytest.mark.parametrize("batch_rows", [1 << 20, 2])
def test_operator_matches_restatement(batch_rows):
    rows = [r for ch in K.NORMAL for r in ch]
    chunks = []
    for ch in K.NORMAL:
        chunks.append(ops.Chunk(*[ops.LongBlock.of(*[r[c] for r in ch]) for c in range(3)]))
    chunks.insert(2, ops.Chunk(*[ops.LongBlock(np.zeros(0, np.int64)) for _ in range(3)]))
    src = ops.MockExec([ops.DataTypes.LongType] * 3, chunks)
    aggs = [ops.RowNumber(), ops.Rank([1]), ops.DenseRank([1]), ops.Sum(2), ops.CountRow()]
    types = [ops.DataTypes.LongType] * 6 + [ops.DataTypes.DecimalType, ops.DataTypes.LongType]
    ex = ops.GpuNonFrameOverWindowExec(src, ops.ExecutionContext(gpu_batch_rows=batch_rows), aggs, [0], [False] * 5, types)
    ex.open()
    out, sizes = [], []
    while True:
        ch = ex.nextChunk()
        if ch is None:
            if ex.produceIsFinished():
                break
            continue
        sizes.append(ch.getPositionCount())
        out.extend(ch.rows())
    assert sizes == [c.getPositionCount() for c in chunks]  # one output chunk per input chunk
    ex.close()
    ex.close()
    cols = [(np.array([0 if r[c] is None else r[c] for r in rows], np.int64), np.array([r[c] is None for r in rows], np.uint8))
            for c in range(3)]
    exp = window_rows([cols], [0], [("ROW_NUMBER", []), ("RANK", [1]), ("DENSE_RANK", [1]), ("SUM", [2]), ("COUNT_STAR", [])])
    assert [r[:3] for r in out] == rows
    assert [list(r[3:]) for r in out] == [list(x) for x in zip(*exp)]


def test_refusals_and_statuses():
    c = ctx()
    T = [N.T_INT64, N.T_FP64, N.T_INT32]

    def status(*a, **k):
        with pytest.raises(N.GsqlError) as e:
            api.Window(c, *a, **k)
        return e.value.status

    assert status(T, [0], [(N.AGG_ROW_NUMBER, []), (N.AGG_SUM, [0])], filter_args=[-1, 0]) == N.E_UNSUPPORTED
    assert status(T, [0], [(N.AGG_FIRST_VALUE, [0])]) == N.E_UNSUPPORTED
    assert status(T, [0], [(N.AGG_AVG_MERGE, [1, 0])]) == N.E_UNSUPPORTED
    assert status(T, [0], [(42, [])]) == N.E_UNSUPPORTED
    assert status(T, [0], [(N.AGG_AVG, [0])]) == N.E_UNSUPPORTED
    assert status(T, [0], [(N.AGG_SUM0, [2])]) == N.E_UNSUPPORTED
    assert status(T + [N.T_DEC128], [0], [(N.AGG_ROW_NUMBER, [])]) == N.E_UNSUPPORTED
    assert status(T, [3], [(N.AGG_ROW_NUMBER, [])]) == N.E_INVALID
    assert status(T, [0], [(N.AGG_RANK, [5])]) == N.E_INVALID
    assert status(T, [0], []) == N.E_INVALID
    spec = N.WindowSpec()  # five RANK columns: the struct holds four, so the count alone is refused
    spec.n_input_cols, spec.npart, spec.ncalls = 1, 0, 1
    spec.calls[0].kind, spec.calls[0].ncols, spec.calls[0].filter_arg = N.AGG_RANK, 5, -1
    import ctypes as C
    h = C.c_void_p()
    assert c.lib.gsql_window_create(c.ptr, C.byref(spec), C.byref(h)) == N.E_UNSUPPORTED
    # the window kinds stay unknown to both aggregations, with the status any unknown kind gets
    for kind in (N.AGG_ROW_NUMBER, N.AGG_RANK, N.AGG_DENSE_RANK):
        for cls in (api.HashAgg, api.SortAgg):
            with pytest.raises(N.GsqlError) as e:
                cls(c, [N.T_INT64], [0], [(kind, [])])
            with pytest.raises(N.GsqlError) as e2:
                cls(c, [N.T_INT64], [0], [(42, [])])
            assert e.value.status == e2.value.status == N.E_UNSUPPORTED
    w = api.Window(c, [N.T_INT64], [0], [(N.AGG_ROW_NUMBER, [])])
    bad = api._alloc_out(c, [N.T_INT64], 4, N.MEM_HOST, [False])
    with pytest.raises(N.GsqlError) as e:
        w.apply([(np.arange(4, dtype=np.int64), None)], out_cols=bad)
    assert e.value.status == N.E_INVALID
    w.close()


def test_profile_names_the_tile_kernel():
    c = ctx()
    c.profile(True)
    c.profile_reset()
    try:
        run([(np.arange(5000, dtype=np.int64) // 7, None)], [0], [("ROW_NUMBER", [])])
        n, ms = c.profile_get("win_tile")
        assert n == 1 and ms > 0
    finally:
        c.profile(False)
