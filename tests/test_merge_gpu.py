"""-m gpu checks of the merge of sorted runs (gsql_merge_*, api.Merge, operators.GpuMergeSortExec, Q3Pipeline.merge_runs)
against the stable merge of tests/merge_ref.py, row for row.  Each case also asserts from the kernel profile which path
ran: the merge-path kernels for images of <= 128 bits, the stable radix sort for wider images, neither for constant keys
or a single non-empty run."""
from collections import Counter

import numpy as np
import pytest

from galaxysql_b200 import api, native as N
from tests import merge_ref as mr
from tests import sort_ref as sr
from tests.golden import merge_kats

pytestmark = pytest.mark.gpu

F64_SPECIALS = np.array([-np.inf, -1.5, -0.0, 0.0, 2.5, np.inf, np.nan], dtype=np.float64)


@pytest.fixture(scope="module")
def ctx():
    from tests import gpu_util
    return gpu_util.ctx()


def _types(cols):
    m = {np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}
    return [m[np.asarray(d).dtype] for d, _ in cols]


def _sorted(cols, keys, desc):
    """One ordered run: the rows of `cols` under the comparator (stable)."""
    p = sr.lexsort_perm(cols, _types(cols), keys, desc)
    return [(d[p], None if nl is None else nl[p]) for d, nl in cols]


def _piece(cols, a, b):
    return [(d[a:b], None if nl is None else nl[a:b]) for d, nl in cols]


def run(ctx, inputs, keys, desc, limit=None, parts=1, mem="host", interleave=False, out_mem=N.MEM_HOST, chunk=None):
    """Consumes every input in `parts` batches (input by input, or round-robin over the inputs) and returns the merged
    rows as numpy columns."""
    from tests import gpu_util
    types = _types(inputs[0])
    m = api.Merge(ctx, types, keys, desc, len(inputs), limit)
    batches = []
    for i, cols in enumerate(inputs):
        n = len(cols[0][0])
        b = np.linspace(0, n, parts + 1).astype(int)
        batches.append([(i, _piece(cols, b[p], b[p + 1])) for p in range(parts) if b[p + 1] > b[p]])
    if interleave:
        order = [x for grp in zip(*[bs + [None] * (max(map(len, batches)) - len(bs)) for bs in batches]) for x in grp if x is not None]
    else:
        order = [x for bs in batches for x in bs]
    for j, (i, piece) in enumerate(order):
        dev = mem == "device" or (mem == "mixed" and j % 2)
        m.consume(i, gpu_util.to_device(piece) if dev else piece)
    total = m.finish()
    outs = []
    while True:
        o = m.next(chunk or max(total, 1), out_mem)
        if len(o[0][0]) == 0:
            break
        outs.append(gpu_util.to_numpy(o))
    m.close()
    if not outs:
        return [(np.zeros(0, np.asarray(d).dtype), np.zeros(0, bool)) for d, _ in inputs[0]]
    return [(np.concatenate([o[c][0] for o in outs]), np.concatenate([o[c][1] for o in outs])) for c in range(len(inputs[0]))]


def check(ctx, inputs, keys, desc, limit=None, path=None, **kw):
    """Runs the merge under the kernel profile and compares it row for row with the stable merge.  path: "merge" (the
    merge-path kernels), "sort" (the stable radix sort: images over 128 bits), "none" (constant keys or at most one
    non-empty run), or None to skip the path check."""
    ctx.profile(True)
    ctx.profile_reset()
    try:
        out = run(ctx, inputs, keys, desc, limit, **kw)
        prof = ctx.profile_dump()
    finally:
        ctx.profile(False)
    want = mr.merged(inputs, _types(inputs[0]), keys, desc, limit)
    mr.assert_rows_equal(out, want)
    if path == "merge":
        assert "k_merge_partition" in prof and "k_merge_tiles" in prof and "k_sort_radix" not in prof, prof
    elif path == "sort":
        assert "k_sort_radix" in prof and "k_merge_tiles" not in prof, prof
    elif path == "none":
        assert "k_sort_radix" not in prof and "k_merge_tiles" not in prof, prof
    check.prof = prof
    return out


def _runs(k, sizes, seed, null_frac=0.05):
    """k ordered runs of (FP64 DESC, INT32 ASC) keys with NULLs and two payload columns (the row's id: input, position)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(k):
        n = int(sizes[i])
        f = np.round(rng.standard_normal(n) * 100, 1)
        sp = rng.random(n) < 0.02
        f[sp] = rng.choice(F64_SPECIALS, int(sp.sum()))
        cols = [(f, rng.random(n) < null_frac), (rng.integers(-5, 5, n).astype(np.int32), rng.random(n) < null_frac),
                (np.full(n, i, np.int64), None), (np.arange(n, dtype=np.int32), None)]
        out.append(_sorted(cols, [0, 1], [True, False]))
    return out


# ------------------------------------------------------------------------------------------------ reference KATs
def _kat_inputs(kat):
    out = []
    for chunks in kat["inputs"]:
        cols = [sum((ch[c] for ch in chunks), []) for c in range(len(kat["types"]))]
        out.append(mr.of_rows(cols, kat["types"]))
    return out


@pytest.mark.parametrize("kat", merge_kats.MERGE_KATS, ids=lambda k: k["name"])
def test_reference_kats_through_api_merge(ctx, kat):
    keys, desc = [c for c, _, _ in kat["order"]], [d for _, d, _ in kat["order"]]
    out = check(ctx, _kat_inputs(kat), keys, desc, kat["offset"] + kat["limit"], path="merge")
    lo, hi = kat["offset"], kat["offset"] + kat["limit"]
    mr.assert_rows_equal([(d[lo:hi], nl[lo:hi]) for d, nl in out], mr.of_rows(kat["expect"], kat["types"]))


@pytest.mark.parametrize("kat", merge_kats.MERGE_KATS, ids=lambda k: k["name"])
def test_reference_kats_through_gpu_merge_sort_exec(ctx, kat):
    from galaxysql_b200 import operators as ops
    T = ops.DataTypes.IntegerType
    srcs = []
    for chunks in kat["inputs"]:
        b = ops.MockExec.builder(T, T)
        for ch in chunks:
            b.withChunk(ops.Chunk(*[ops.IntegerBlock.of(*col) for col in ch]))
        srcs.append(b.build())
    orders = [ops.OrderByOption(c, ops.Direction.DESCENDING if d else ops.Direction.ASCENDING, nd) for c, d, nd in kat["order"]]
    exec_ = ops.GpuMergeSortExec(srcs, orders, kat["offset"], kat["limit"], ops.ExecutionContext(chunk_size=3))
    rows = [r for ch in ops.SingleExecTest(exec_).exec().result() for r in ch.rows()]
    assert rows == list(zip(*kat["expect"]))


def test_gpu_merge_sort_exec_resumes_after_blocked_inputs_and_skips(ctx):
    from galaxysql_b200 import operators as ops
    from tests.test_merge_cpu import _Blocking
    T = ops.DataTypes.LongType
    runs = [np.sort(np.random.default_rng(i).integers(0, 50, 40)) for i in range(3)]
    srcs = [_Blocking([T], [ops.Chunk(ops.LongBlock(r[j:j + 7].astype(np.int64))) for j in range(0, 40, 7)]) for r in runs]
    exec_ = ops.GpuMergeSortExec(srcs, [ops.OrderByOption(0)], 5, 60, ops.ExecutionContext(chunk_size=8, gpu_batch_rows=10))
    exec_.open()
    got, nones = [], 0
    while True:
        ch = exec_.nextChunk()
        if ch is None:
            if exec_.produceIsFinished():
                break
            nones += 1
            continue
        got += [r[0] for r in ch.rows()]
    exec_.close()
    assert nones > 0
    assert got == sorted(np.concatenate(runs).tolist())[5:65]


# ------------------------------------------------------------------------------------------------ input shapes
@pytest.mark.parametrize("k", [1, 2, 3, 7, 8, 64, 1000, 4096])
def test_k_inputs(ctx, k):
    rng = np.random.default_rng(k)
    sizes = rng.integers(0, max(2, 400_000 // k), k)
    sizes[rng.random(k) < 0.1] = 0  # some empty inputs
    sizes[0] = max(sizes[0], 1)
    inputs = _runs(k, sizes, k)
    nonempty = int((sizes > 0).sum())
    check(ctx, inputs, [0, 1], [True, False], path="merge" if nonempty > 1 else "none")
    check(ctx, inputs, [0, 1], [True, False], limit=1000, path="merge" if nonempty > 1 else "none")


def test_empty_inputs(ctx):
    empty = _runs(1, [0], 1)[0]
    check(ctx, [empty, empty, empty], [0, 1], [True, False], path="none")
    one = _runs(1, [1000], 2)[0]
    check(ctx, [empty, one, empty], [0, 1], [True, False], path="none")


def test_one_row_inputs_next_to_ten_million(ctx):
    rng = np.random.default_rng(3)
    n = 10_000_000
    big = _sorted([(rng.integers(-1 << 40, 1 << 40, n), None), (np.arange(n, dtype=np.int32), None)], [0], [False])
    one = [[(np.array([v], np.int64), None), (np.array([-1 - i], np.int32), None)] for i, v in enumerate((int(big[0][0][n // 2]), -(1 << 41), 1 << 41))]
    check(ctx, [one[0], big, one[1], one[2]], [0], [False], path="merge")


@pytest.mark.parametrize("mem", ["host", "device", "mixed"])
def test_interleaved_chunks_and_mixed_batches(ctx, mem):
    inputs = _runs(5, [30_000, 1, 0, 50_000, 7777], 4)
    check(ctx, inputs, [0, 1], [True, False], parts=6, mem=mem, interleave=True, path="merge")
    check(ctx, inputs, [0, 1], [True, False], limit=500, parts=6, mem=mem, interleave=True, path="merge",
          out_mem=N.MEM_DEVICE, chunk=77)


def test_misaligned_device_views(ctx):
    import torch
    inputs = _runs(3, [10_001, 5_003, 7_007], 5)
    for off in (1, 3):
        views = []
        for cols in inputs:
            dv = []
            for d, nl in cols:
                td = torch.from_numpy(np.ascontiguousarray(d)).cuda()[off:]
                tn = None if nl is None else torch.from_numpy(nl.astype(np.uint8)).cuda()[off:]
                dv.append((td, tn))
            views.append(dv)
        m = api.Merge(ctx, _types(inputs[0]), [0, 1], [True, False], 3)
        for i, v in enumerate(views):
            m.consume(i, v)
        from tests import gpu_util
        out = gpu_util.to_numpy(m.result(N.MEM_DEVICE))
        m.close()
        mr.assert_rows_equal(out, mr.merged([_piece(c, off, None) for c in inputs], _types(inputs[0]), [0, 1], [True, False]))


# ------------------------------------------------------------------------------------------------ key types and images
@pytest.mark.parametrize("dtype", [np.int32, np.int64, np.float64], ids=["int32", "int64", "fp64"])
@pytest.mark.parametrize("desc", [False, True])
def test_key_types_with_nulls_and_special_values(ctx, dtype, desc):
    rng = np.random.default_rng(7)
    if dtype == np.float64:
        pool = F64_SPECIALS
    else:
        info = np.iinfo(dtype)
        pool = np.array([info.min, info.min + 1, -1, 0, 1, info.max - 1, info.max], dtype=dtype)
    inputs = []
    for i in range(6):
        n = 2000 + 100 * i
        cols = [(rng.choice(pool, n).astype(dtype), rng.random(n) < 0.1), (np.arange(n, dtype=np.int64), None)]
        inputs.append(_sorted(cols, [0], [desc]))
    check(ctx, inputs, [0], [desc], path="merge")  # row for row, by raw bits: -0.0 before +0.0, NaN above +Inf


@pytest.mark.parametrize("width", ["u32", "u64", "k128", "over128", "constant"])
def test_image_widths(ctx, width):
    rng = np.random.default_rng(8)
    n, k = 60_000, 5
    inputs = []
    for i in range(k):
        if width == "u32":
            cols = [(rng.integers(-1000, 1000, n).astype(np.int32), None)]
            keys = [0]
        elif width == "u64":
            cols = [(rng.integers(-1 << 40, 1 << 40, n), None)]
            keys = [0]
        elif width in ("k128", "over128"):
            nk = 2 if width == "k128" else 3
            cols = [(rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, endpoint=True, dtype=np.int64), None)
                    for _ in range(nk)]
            for c in range(nk):
                cols[c][0][:2] = [np.iinfo(np.int64).min, np.iinfo(np.int64).max]  # full-range keys: 64 bits each
            keys = list(range(nk))
        else:
            cols = [(np.full(n, 42, np.int64), None)]
            keys = [0]
        cols.append((np.arange(n, dtype=np.int32) + i * n, None))
        inputs.append(_sorted(cols, keys, [False] * len(keys)))
    path = {"u32": "merge", "u64": "merge", "k128": "merge", "over128": "sort", "constant": "none"}[width]
    check(ctx, inputs, keys, [bool(j % 2) for j in range(len(keys))] if width == "constant" else [False] * len(keys), path=path)
    if width in ("k128", "over128"):
        check(ctx, inputs, keys, [False] * len(keys), limit=777, path=path)


# ------------------------------------------------------------------------------------------------ limits
@pytest.mark.parametrize("limit_of", [lambda t, m: 0, lambda t, m: 1, lambda t, m: m // 2, lambda t, m: t + 5],
                         ids=["0", "1", "within_one_input", "above_total"])
def test_limits(ctx, limit_of):
    inputs = _runs(6, [10_000, 3, 20_000, 0, 5_000, 12_345], 9)
    total = sum(len(c[0][0]) for c in inputs)
    limit = limit_of(total, 5_000)
    check(ctx, inputs, [0, 1], [True, False], limit=limit, path="none" if limit == 0 else "merge")


def test_rows_past_an_inputs_quota_are_dropped(ctx):
    """Input 0 holds L ordered rows and then rows that would lead the output: past its quota, the merge must drop them."""
    L = 100
    a = [(np.arange(L, dtype=np.int64) + 1000, None), (np.zeros(L, np.int32), None)]
    tail = [(np.arange(50, dtype=np.int64) - 1000, None), (np.ones(50, np.int32), None)]
    b = [(np.arange(0, 3 * L, 3, dtype=np.int64) + 1000, None), (np.full(L, 2, np.int32), None)]
    m = api.Merge(ctx, [N.T_INT64, N.T_INT32], [0], [False], 2, L)
    m.consume(0, a)
    m.consume(1, b)
    m.consume(0, tail)
    out = m.result()
    m.close()
    assert len(out[0][0]) == L and not out[1][0].tolist().count(1)
    mr.assert_rows_equal(out, mr.merged([a, b], [N.T_INT64, N.T_INT32], [0], [False], L))


# ------------------------------------------------------------------------------------------------ unsorted inputs
@pytest.mark.parametrize("k", [2, 5])
def test_unsorted_inputs_come_out_as_the_input_multiset(ctx, k):
    rng = np.random.default_rng(10 + k)
    inputs = [[(rng.integers(-100, 100, 20_000 + i), rng.random(20_000 + i) < 0.1), (np.arange(20_000 + i, dtype=np.int32), None)]
              for i in range(k)]
    out = run(ctx, inputs, [0], [False])
    cat = mr.concat(inputs)
    assert Counter(map(bytes, sr.row_matrix(out))) == Counter(map(bytes, sr.row_matrix(cat)))


# ------------------------------------------------------------------------------------------------ errors
def test_argument_and_state_errors(ctx):
    for n in (0, N.MAX_MERGE_INPUTS + 1, -1):
        with pytest.raises(N.GsqlError) as e:
            api.Merge(ctx, [N.T_INT64], [0], [False], n)
        assert e.value.status == N.E_INVALID
    with pytest.raises(N.GsqlError) as e:
        api.Merge(ctx, [N.T_INT64, N.T_DEC128], [0], [False], 2)
    assert e.value.status == N.E_UNSUPPORTED
    with pytest.raises(N.GsqlError) as e:
        api.Merge(ctx, [N.T_INT64], [0], [False], 2, limit=-2)
    assert e.value.status == N.E_INVALID
    m = api.Merge(ctx, [N.T_INT64], [0], [False], N.MAX_MERGE_INPUTS)
    for bad in (-1, N.MAX_MERGE_INPUTS):
        with pytest.raises(N.GsqlError) as e:
            m.consume(bad, [(np.array([1], np.int64), None)])
        assert e.value.status == N.E_INVALID
    m.consume(N.MAX_MERGE_INPUTS - 1, [(np.array([1, 2], np.int64), None)])
    assert m.finish() == 2
    with pytest.raises(N.GsqlError) as e:
        m.consume(0, [(np.array([1], np.int64), None)])
    assert e.value.status == N.E_STATE
    m.close()


# ------------------------------------------------------------------------------------------------ size
def test_100m_rows_in_8_inputs(ctx):
    import torch
    k, per = 8, 12_500_000
    g = torch.Generator(device="cuda").manual_seed(12)

    def order(f, i):  # stable: INT32 ASC, then FP64 DESC
        p = torch.sort(i, stable=True).indices
        q = torch.sort(f[p], descending=True, stable=True).indices
        return p[q]
    runs, fs, is_, ids = [], [], [], []
    for r in range(k):
        f = torch.randint(-(1 << 20), 1 << 20, (per,), device="cuda", generator=g).double() / 8.0
        i = torch.randint(-(1 << 15), 1 << 15, (per,), device="cuda", generator=g, dtype=torch.int32)
        p = order(f, i)
        rid = torch.arange(r * per, (r + 1) * per, device="cuda", dtype=torch.int64)[p]
        runs.append([(f[p], None), (i[p], None), (rid, None), (rid.double(), None)])
        fs.append(f[p])
        is_.append(i[p])
        ids.append(rid)
    torch.cuda.synchronize()  # the library reads the runs on its own stream
    m = api.Merge(ctx, [N.T_FP64, N.T_INT32, N.T_INT64, N.T_FP64], [0, 1], [True, False], k)
    ctx.profile(True)
    ctx.profile_reset()
    for r in range(k):
        m.consume(r, runs[r])
    out = m.result(N.MEM_DEVICE, nullable_out=False)
    prof = ctx.profile_dump()
    ctx.profile(False)
    m.close()
    assert "k_merge_tiles" in prof and "k_sort_radix" not in prof, prof
    F, I, R = torch.cat(fs), torch.cat(is_), torch.cat(ids)
    want = R[order(F, I)]
    assert torch.equal(out[2][0], want)
    assert torch.equal(out[3][0], want.double())


# ------------------------------------------------------------------------------------------------ Q3
@pytest.mark.parametrize("limit", [None, 10])
@pytest.mark.parametrize("k", [3, 8])
def test_q3_rank0_merge_with_simulated_ranks(ctx, limit, k):
    from galaxysql_b200 import pipelines
    from tests import gpu_util as gu
    from tests import q3_util
    tables = q3_util.q3_tables(0, 1, ncust=8000, nord=60000, nline=220000)
    q3 = pipelines.Q3Pipeline(ctx, customer_capacity=8000, orders_capacity=60000, lineitem_capacity=220000, nslabs=3,
                              expected_groups=4096, limit=limit)
    q3.order_by = False  # the groups unordered; _sorted / merge_runs below keep the pipeline's limit
    groups = q3.run(gu.to_device(tables[0]), gu.to_device(tables[1]), gu.to_device(tables[2]))
    n = int(groups[0][0].shape[0])
    bounds = np.linspace(0, n, k + 1).astype(int)
    runs = [q3._sorted([(d[bounds[r]:bounds[r + 1]], None if nl is None else nl[bounds[r]:bounds[r + 1]]) for d, nl in groups])
            for r in range(k)]
    ctx.profile(True)
    ctx.profile_reset()
    out = gu.to_numpy(q3.merge_runs(runs))
    prof = ctx.profile_dump()
    ctx.profile(False)
    q3.close()
    assert "k_merge_tiles" in prof and "k_sort_radix" not in prof, prof
    types, keys, desc = q3.Q3_OUT_TYPES, [3, 1], [True, False]
    mr.assert_rows_equal(out, mr.merged([gu.to_numpy(r) for r in runs], types, keys, desc, limit))
    whole = gu.to_numpy(groups)
    single = gu.to_numpy(q3._sorted(groups))
    sr.check_ordered(out, whole, types, keys, desc, limit)
    assert np.array_equal(sr.key_matrix(out, types, keys), sr.key_matrix(single, types, keys))
    exp = q3_util.q3_oracle(*tables)
    ref = [(c[0], None) for c in exp]
    if limit is not None:
        p = sr.lexsort_perm(ref, types, keys, desc)[:limit]
        ref = [(c[0][p], None) for c in ref]
    gu.approx_rows_equal(out, ref, float_cols=[3], key_cols=[0, 1, 2], rtol=1e-6)
