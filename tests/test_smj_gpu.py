"""gsql_smj on the GPU against the SortMergeJoinExec restatement (tests/smj_ref.py), row for row and in order, through
api.SortMergeJoin and operators.GpuSortMergeJoinExec: every join type, single joins, anti operands, 1-8 mixed keys under
ASC / DESC with NULLs, signed zeros, NaN payloads and integer extremes, run lengths around the tile, batch splits, device
batches, every error, and the composition with gsql_sort, gsql_join, gsql_sortagg and gsql_agg."""
import ctypes as C
import functools
import struct
from collections import Counter

import numpy as np
import pytest

from galaxysql_b200 import api, native as N, operators as ops
from tests import smj_ref as ref
from tests.gpu_util import ctx, to_device
from tests.golden.smj_kats import SMJ_KATS, encode
from tests.test_smj_cpu import kat_ref, kat_rows

pytestmark = pytest.mark.gpu

TILE = 1024  # SJ_TILE of smj.cuh
NP = {N.T_INT32: np.int32, N.T_INT64: np.int64, N.T_FP64: np.float64}
JT = {ref.INNER: N.JOIN_INNER, ref.LEFT: N.JOIN_LEFT, ref.RIGHT: N.JOIN_RIGHT, ref.SEMI: N.JOIN_SEMI, ref.ANTI: N.JOIN_ANTI}
UNIFIED = {N.T_INT32: "int", N.T_INT64: "int", N.T_FP64: "double"}


def _canon(v):
    if v is None:
        return None
    if isinstance(v, float):
        return ("f", struct.unpack("<q", struct.pack("<d", v))[0])
    return int(v)


def cols_to_rows(cols):
    if not cols:
        return []
    n = len(cols[0][0])
    vals = []
    for d, nl in cols:
        d = d.cpu().numpy() if hasattr(d, "cpu") else np.asarray(d)
        nl = None if nl is None else (nl.cpu().numpy() if hasattr(nl, "cpu") else np.asarray(nl))
        vals.append([None if nl is not None and nl[r] else d[r].item() for r in range(n)])
    return [tuple(_canon(c[r]) for c in vals) for r in range(n)]


def rows_to_cols(rows, types):
    cols = []
    for j, t in enumerate(types):
        vals = [r[j] for r in rows]
        nl = np.array([v is None for v in vals], bool)
        cols.append((np.array([0 if v is None else v for v in vals], dtype=NP[t]), nl if nl.any() else None))
    return cols


def canon_rows(rows):
    return [tuple(_canon(v) for v in r) for r in rows]


def gpu_join(outer, inner, otypes, itypes, jt, okeys, ikeys, ktypes, desc=None, single=False, anti=None,
             inner_splits=(), outer_splits=(), mem="host", max_rows=None):
    """Runs gsql_smj over row lists cut at the splits; returns the output rows in order."""
    j = api.SortMergeJoin(ctx(), JT[jt], otypes, itypes, okeys, ikeys, ktypes, desc=desc, max_one_row=single,
                          anti_operands=anti)
    try:
        cuts = [0] + list(inner_splits) + [len(inner)]
        for a, b in zip(cuts[:-1], cuts[1:]):
            part = rows_to_cols(inner[a:b], itypes)
            j.inner_consume(to_device(part) if mem == "device" else part)
        j.inner_finish()
        out = []
        cuts = [0] + list(outer_splits) + [len(outer)]
        for a, b in zip(cuts[:-1], cuts[1:]):
            part = rows_to_cols(outer[a:b], otypes)
            n = j.probe(to_device(part) if mem == "device" else part)
            got = 0
            while True:
                cols = j.next(max_rows or max(n, 1), N.MEM_DEVICE if mem == "device" else N.MEM_HOST)
                rows = cols_to_rows(cols)
                if not rows:
                    break
                got += len(rows)
                out += rows
            assert got == n
        return out
    finally:
        j.close()


def ref_join(outer, inner, otypes, itypes, jt, okeys, ikeys, ktypes, desc=None, single=False, anti=None):
    asc = None if desc is None else [not d for d in desc]
    return canon_rows(ref.smj_ref(outer, inner, jt, okeys, ikeys, [UNIFIED[t] for t in ktypes], ascending=asc,
                                  max_one_row=single, anti_operands=anti, n_inner_cols=len(itypes)))


def sort_rows(rows, keys, ktypes, desc):
    def cmp(a, b):
        for k, c in enumerate(keys):
            x = ref.number_compare(a[c], b[c], UNIFIED[ktypes[k]]) * (-1 if desc[k] else 1)
            if x:
                return x
        return 0
    return sorted(rows, key=functools.cmp_to_key(cmp))


VALUES = {
    N.T_INT32: [np.iinfo(np.int32).min, -7, -1, 0, 1, 2, 3, 5, np.iinfo(np.int32).max],
    N.T_INT64: [np.iinfo(np.int64).min, -(1 << 40), -1, 0, 1, 2, 3, 1 << 40, np.iinfo(np.int64).max],
    N.T_FP64: [float("-inf"), -2.5, -0.0, 0.0, 1.0, 2.0, 3.0, float("inf"), float("nan"),
               struct.unpack("<d", struct.pack("<q", 0x7ff0000000000123))[0]],  # a NaN with its own payload
}


def random_side(rng, n, types, keys, domain, null_rate, desc, ktypes):
    rows = []
    pools = {c: list(VALUES[t][:domain]) for c, t in enumerate(types)}
    for _ in range(n):
        row = []
        for c, t in enumerate(types):
            if rng.random() < null_rate:
                row.append(None)
            else:
                v = pools[c][rng.integers(len(pools[c]))]
                row.append(float(v) if t == N.T_FP64 else int(v))
        rows.append(tuple(row))
    return sort_rows(rows, keys, ktypes, desc)


def key_types_for(otypes, itypes, okeys, ikeys):
    out = []
    for o, i in zip(okeys, ikeys):
        a, b = otypes[o], itypes[i]
        out.append(N.T_FP64 if N.T_FP64 in (a, b) else (N.T_INT64 if N.T_INT64 in (a, b) else N.T_INT32))
    return out


def ordered(rows, keys):  # the sort is stable: ordered rows are their own sorted order
    return rows == sort_rows(rows, keys, [N.T_INT32] * len(keys), [False] * len(keys))


# ------------------------------------------------------------------------------------------------ known answers
@pytest.mark.parametrize("case", SMJ_KATS, ids=lambda c: c["name"])
def test_kats_through_the_api_and_the_operator(case):
    case = encode(case)
    outer, inner = kat_rows(case, "outer"), kat_rows(case, "inner")
    ot, it = [N.T_INT32] * len(case["outer_types"]), [N.T_INT32] * len(case["inner_types"])
    okeys, ikeys = [k[0] for k in case["keys"]], [k[1] for k in case["keys"]]
    kt = [N.T_INT32] * len(okeys)
    if case["cond"] is not None:  # any other condition keeps the stock operator
        with pytest.raises(N.GsqlError) as e:
            api.SortMergeJoin(ctx(), JT[case["join"]], ot, it, okeys, ikeys, kt, max_one_row=case["single"],
                              cond_ne=[(0, 0)])
        assert e.value.status == N.E_UNSUPPORTED
        return
    if not (ordered(outer, okeys) and ordered(inner, ikeys)):
        # the reference's anti-join cases feed an inner side that is not ordered (1 2 3 4 | 3 4 5 6): the stock walk gives
        # an answer there, gsql_smj an error naming the side
        with pytest.raises(N.GsqlError, match="inner") as e:
            gpu_join(outer, inner, ot, it, case["join"], okeys, ikeys, kt, single=case["single"], anti=case["anti"])
        assert e.value.status == N.E_INVALID
        return
    if case["expect"] is None:
        with pytest.raises(N.MoreThanOneRowError):
            gpu_join(outer, inner, ot, it, case["join"], okeys, ikeys, kt, single=case["single"], anti=case["anti"])
    else:
        got = gpu_join(outer, inner, ot, it, case["join"], okeys, ikeys, kt, single=case["single"], anti=case["anti"],
                       outer_splits=[4] if len(outer) > 4 else [])
        assert got == canon_rows(kat_ref(case))
        assert Counter(got) == Counter(canon_rows(zip(*case["expect"])) if case["expect"][0] else [])
    # the operator over the reference's own chunks
    I = ops.DataTypes.IntegerType

    def mock(side):
        chunks = [ops.Chunk(*[ops.IntegerBlock.of(*col) for col in ch]) for ch in case[side]]
        return ops.MockExec([I] * len(case[side + "_types"]), chunks)

    keys = [ops.EquiJoinKey(o, i, I) for o, i in case["keys"]]
    ex = ops.GpuSortMergeJoinExec(mock("outer"), mock("inner"), JT[case["join"]], case["single"], keys, [True] * len(keys),
                                  None, case["anti"], ops.ExecutionContext(chunk_size=3, gpu_batch_rows=5))
    if case["expect"] is None:
        with pytest.raises(ops.TddlRuntimeException):
            ops.SingleExecTest(ex).exec()
        return
    rows = [tuple(_canon(v) for v in r) for ch in ops.SingleExecTest(ex).exec().result() for r in ch.rows()]
    assert rows == canon_rows(kat_ref(case))


# ------------------------------------------------------------------------------------------------ semantics, random
CASES = [(jt, single, anti) for jt in (ref.INNER, ref.LEFT, ref.RIGHT, ref.SEMI, ref.ANTI)
         for single in ((False, True) if jt in (ref.INNER, ref.LEFT) else (False,))
         for anti in (((None, [1]) if jt == ref.ANTI else (None,)))]


@pytest.mark.parametrize("jt,single,anti", CASES)
@pytest.mark.parametrize("seed", range(6))
def test_random_ordered_inputs(jt, single, anti, seed):
    rng = np.random.default_rng(seed * 31 + len(jt))
    nk = [1, 2, 3, 8, 5, 1][seed]
    all_t = [N.T_INT32, N.T_INT64, N.T_FP64]
    otypes = [all_t[rng.integers(3)] for _ in range(nk)] + [N.T_INT64, N.T_INT32]
    itypes = [otypes[k] if rng.random() < 0.6 else all_t[rng.integers(3)] for k in range(nk)] + [N.T_INT64, N.T_FP64]
    keys = list(range(nk))
    kt = key_types_for(otypes, itypes, keys, keys)
    desc = [bool(rng.random() < 0.5) for _ in range(nk)]
    domain = int(rng.choice([2, 4, 9])) if nk < 4 else 2
    null_rate = float(rng.choice([0.0, 0.05, 0.2]))
    outer = random_side(rng, int(rng.integers(0, 3 * TILE)), otypes, keys, domain, null_rate, desc, kt)
    inner = random_side(rng, int(rng.integers(0, 2 * TILE)), itypes, keys, domain, null_rate, desc, kt)
    if single:  # one inner row per key, so that most cases do not raise
        seen, uniq = set(), []
        for r in inner:
            k = tuple(_canon(r[c]) for c in keys)
            if k not in seen:
                seen.add(k)
                uniq.append(r)
        inner = uniq
    args = (outer, inner, otypes, itypes, jt, keys, keys, kt)
    try:
        want = ref_join(*args, desc=desc, single=single, anti=anti)
    except ref.MoreThanOneRow:
        with pytest.raises(N.MoreThanOneRowError):
            gpu_join(*args, desc=desc, single=single, anti=anti)
        return
    splits = sorted(set(int(x) for x in rng.integers(0, len(outer) + 1, 3)))
    got = gpu_join(*args, desc=desc, single=single, anti=anti, outer_splits=splits, inner_splits=[len(inner) // 2],
                   max_rows=int(rng.choice([7, 1000, 1 << 20])))
    assert got == want


@pytest.mark.parametrize("run", [1, 2, TILE - 1, TILE, TILE + 1])
@pytest.mark.parametrize("jt", [ref.INNER, ref.LEFT, ref.SEMI, ref.ANTI])
def test_run_lengths_around_the_tile(run, jt):
    n = 6 * TILE + 3
    inner = [(k // run, k) for k in range(0, n, 2)]
    outer = [(k // run, -k) for k in range(n) if k % 3]
    t = [N.T_INT64, N.T_INT64]
    assert gpu_join(outer, inner, t, t, jt, [0], [0], [N.T_INT64]) == ref_join(outer, inner, t, t, jt, [0], [0], [N.T_INT64])


def test_one_inner_run_of_ten_million_rows():
    n = 10_000_000
    j = api.SortMergeJoin(ctx(), N.JOIN_LEFT, [N.T_INT64], [N.T_INT64, N.T_INT32], [0], [0])
    try:
        j.inner_consume([(np.r_[np.full(n, 5, np.int64), [9]], None), (np.arange(n + 1, dtype=np.int32), None)])
        j.inner_finish()
        assert j.probe([(np.array([4, 5, 5, 6, 9], np.int64), None)]) == 1 + 2 * n + 1 + 1
        (o, onl), (k, knl), (v, vnl) = j.next(2 * n + 3)
        assert j.next(1)[0][0].shape[0] == 0
    finally:
        j.close()
    assert o.tolist()[:2] == [4, 5] and o[-2:].tolist() == [6, 9] and knl[0] and knl[-2] and not knl[1:-2].any()
    assert np.array_equal(v[1:1 + n], np.arange(n)) and np.array_equal(v[1 + n:1 + 2 * n], np.arange(n)) and v[-1] == n


def test_many_to_many_beyond_two_to_the_32_rows_counts_exactly():
    m = 70_000  # one outer run and one inner run of m rows: m * m > 2^32 output rows
    j = api.SortMergeJoin(ctx(), N.JOIN_INNER, [N.T_INT32], [N.T_INT32], [0], [0])
    try:
        j.inner_consume([(np.r_[np.zeros(m, np.int32), [1]].astype(np.int32), None)])
        j.inner_finish()
        total = j.probe([(np.r_[[-1], np.zeros(m, np.int32), [1, 2]].astype(np.int32), None)])
        assert total == m * m + 1 and total > 1 << 32
        first = cols_to_rows(j.next(5))
        assert first == [(0, 0)] * 5
    finally:
        j.close()


def test_signed_zeros_nan_and_unified_integer_keys():
    outer = [(-1,), (0,), (2,), (3,)]
    inner = [(-1.0, 1), (-0.0, 2), (0.0, 3), (2.0, 4), (2.5, 5), (float("nan"), 6)]
    t_o, t_i = [N.T_INT32], [N.T_FP64, N.T_INT32]
    got = gpu_join(outer, inner, t_o, t_i, ref.INNER, [0], [0], [N.T_FP64])
    assert got == ref_join(outer, inner, t_o, t_i, ref.INNER, [0], [0], [N.T_FP64])
    assert got == [(-1, _canon(-1.0), 1), (0, _canon(0.0), 3), (2, _canon(2.0), 4)]  # 0 converts to +0.0 only
    nans = [(float("nan"), 1), (VALUES[N.T_FP64][-1], 2)]  # different NaN payloads are one value
    got = gpu_join([(VALUES[N.T_FP64][-1],)], nans, [N.T_FP64], [N.T_FP64, N.T_INT32], ref.INNER, [0], [0], [N.T_FP64])
    assert [r[2] for r in got] == [1, 2] and got[0][1] == _canon(float("nan"))


def test_desc_not_in_misses_a_null_that_is_not_first():
    t = [N.T_INT32]
    outer, inner = [(5,), (3,), (1,)], [(4,), (2,), (None,)]
    assert gpu_join(outer, inner, t, t, ref.ANTI, [0], [0], t, desc=[True], anti=[0]) == [(5,), (3,), (1,)]
    assert gpu_join(outer[::-1], inner[::-1], t, t, ref.ANTI, [0], [0], t, anti=[0]) == []


@pytest.mark.parametrize("mem", ["host", "device"])
def test_every_outer_split_and_inner_batches_of_one_row(mem):
    t = [N.T_INT32, N.T_INT64]
    outer = sort_rows([(k % 7 if k % 5 else None, k) for k in range(23)], [0], [N.T_INT32], [False])
    inner = sort_rows([(k % 9, -k) for k in range(15)], [0], [N.T_INT32], [False])
    want = ref_join(outer, inner, t, t, ref.LEFT, [0], [0], [N.T_INT32])
    for s in range(len(outer) + 1):
        got = gpu_join(outer, inner, t, t, ref.LEFT, [0], [0], [N.T_INT32], outer_splits=[s], mem=mem,
                       inner_splits=list(range(1, len(inner))), max_rows=1 if s % 2 else 7)
        assert got == want


def test_empty_sides_and_empty_batches():
    t = [N.T_INT64]
    for jt in (ref.INNER, ref.LEFT, ref.ANTI):
        assert gpu_join([(1,), (2,)], [], t, t, jt, [0], [0], t, inner_splits=[0, 0]) == ref_join([(1,), (2,)], [], t, t, jt, [0], [0], t)
        assert gpu_join([], [(1,)], t, t, jt, [0], [0], t, outer_splits=[0]) == []


def test_misaligned_device_slices():
    import torch
    k = np.repeat(np.arange(3000, dtype=np.int32), 2)
    dk = torch.from_numpy(np.r_[np.zeros(1, np.int32), k]).cuda()[1:]
    dv = torch.from_numpy(np.r_[np.zeros(1, np.int32), np.arange(6000, dtype=np.int32)]).cuda()[1:]
    inner = dk[::2].contiguous()[1:]
    torch.cuda.synchronize()  # the library's stream does not wait for torch's
    j = api.SortMergeJoin(ctx(), N.JOIN_INNER, [N.T_INT32, N.T_INT32], [N.T_INT32], [0], [0])
    try:
        j.inner_consume([(inner, None)])
        j.inner_finish()
        n = j.probe([(dk, None), (dv, None)])
        got = j.next(n, N.MEM_DEVICE)
        assert j.next(1, N.MEM_DEVICE)[0][0].shape[0] == 0
    finally:
        j.close()
    assert n == 6000 - 2
    assert np.array_equal(got[1][0].cpu().numpy(), np.arange(2, 6000, dtype=np.int32))


# ------------------------------------------------------------------------------------------------ errors
def _smj(jt=N.JOIN_INNER, **kw):
    return api.SortMergeJoin(ctx(), jt, [N.T_INT64, N.T_INT64], [N.T_INT64], [0], [0], **kw)


def test_unordered_inputs_are_errors():
    j = _smj()
    j.inner_consume([(np.array([1, 3, 2], np.int64), None)])
    with pytest.raises(N.GsqlError, match="inner") as e:
        j.inner_finish()
    assert e.value.status == N.E_INVALID
    j.close()
    for desc, rows in ((False, [[3, 1]]), (False, [[1, 5], [4, 6]]), (True, [[5, 4], [6]])):
        j = _smj(desc=[desc])
        j.inner_consume([(np.array([1, 2, 3] if not desc else [3, 2, 1], np.int64), None)])
        j.inner_finish()
        with pytest.raises(N.GsqlError, match="outer") as e:
            for r in rows:
                j.probe([(np.array(r, np.int64), None), (np.zeros(len(r), np.int64), None)])
                while j.next(100)[0][0].shape[0]:
                    pass
        assert e.value.status == N.E_INVALID
        j.close()


def test_single_join_violation_surfaces_at_the_probe():
    j = _smj(N.JOIN_LEFT, max_one_row=True)
    j.inner_consume([(np.array([1, 2, 2], np.int64), None)])
    j.inner_finish()
    assert j.probe([(np.array([1], np.int64), None), (np.zeros(1, np.int64), None)]) == 1
    j.next(10)
    j.next(10)
    with pytest.raises(N.MoreThanOneRowError):
        j.probe([(np.array([2], np.int64), None), (np.zeros(1, np.int64), None)])
    j.close()


@pytest.mark.parametrize("kw,jt", [(dict(cond_ne=[(0, 1)]), N.JOIN_INNER), (dict(build_outer=True), N.JOIN_INNER),
                                   (dict(max_one_row=True), N.JOIN_SEMI), (dict(max_one_row=True), N.JOIN_ANTI),
                                   (dict(max_one_row=True), N.JOIN_RIGHT)])
def test_refused_specs(kw, jt):
    with pytest.raises(N.GsqlError) as e:
        _smj(jt, **kw)
    assert e.value.status == N.E_UNSUPPORTED


def test_refused_types_and_key_counts():
    for ot, it in (([N.T_DEC128], [N.T_INT64]), ([N.T_INT64], [N.T_DEC128])):
        with pytest.raises(N.GsqlError) as e:
            api.SortMergeJoin(ctx(), N.JOIN_INNER, ot, it, [0], [0], [N.T_INT64])
        assert e.value.status == N.E_UNSUPPORTED
    s = api._join_spec(N.JOIN_INNER, [N.T_INT64], [N.T_INT64], [0], [0], None, False, False, None, ())
    for nk in (0, N.MAX_KEYS + 1):
        s.nkeys = nk
        h = C.c_void_p()
        assert ctx().lib.gsql_smj_create(ctx().ptr, C.byref(s), (C.c_int32 * 16)(), C.byref(h)) == N.E_UNSUPPORTED


def test_an_outer_batch_of_two_to_the_31_minus_one_rows_is_refused():
    import torch
    keys = torch.zeros((1 << 31) - 1, dtype=torch.int32, device="cuda")  # real rows: nothing is read past them
    torch.cuda.synchronize()
    j = api.SortMergeJoin(ctx(), N.JOIN_INNER, [N.T_INT32], [N.T_INT32], [0], [0])
    try:
        j.inner_consume([(np.zeros(1, np.int32), None)])
        j.inner_finish()
        with pytest.raises(N.CapacityError):  # its n + 1 output offsets would overflow the scan's 32-bit item count
            j.probe([(keys, None)])
    finally:
        j.close()
    del keys
    torch.cuda.empty_cache()


def test_call_order_and_missing_nulls_buffer():
    j = _smj(N.JOIN_LEFT)
    with pytest.raises(N.GsqlError) as e:
        j.probe([(np.array([1], np.int64), None), (np.zeros(1, np.int64), None)])
    assert e.value.status == N.E_STATE
    j.inner_consume([(np.array([1], np.int64), None)])
    j.inner_finish()
    with pytest.raises(N.GsqlError) as e:
        j.inner_consume([(np.array([2], np.int64), None)])
    assert e.value.status == N.E_STATE
    assert j.probe([(np.array([1, 2], np.int64), None), (np.zeros(2, np.int64), None)]) == 2
    with pytest.raises(N.GsqlError) as e:
        j.probe([(np.array([3], np.int64), None), (np.zeros(1, np.int64), None)])
    assert e.value.status == N.E_STATE
    with pytest.raises(N.GsqlError) as e:  # row 2 is NULL-padded: the inner column needs a nulls buffer
        j.next(2, nullable_out=False)
    assert e.value.status == N.E_INVALID
    assert cols_to_rows(j.next(2)) == [(1, 0, 1), (2, 0, None)]  # the cursor did not move
    j.close()


# ------------------------------------------------------------------------------------------------ composition
def _sorted_by_gpu(cols, keys, desc):
    s = api.Sort(ctx(), [N.T_INT64] * len(cols), keys, desc)
    s.consume(cols)
    out = s.result()
    s.close()
    return out


def test_sort_then_smj_equals_the_hash_join_and_is_ordered():
    rng = np.random.default_rng(7)
    n = 300_000
    o = [(rng.integers(0, 50_000, n).astype(np.int64), None), (np.arange(n, dtype=np.int64), None)]
    i = [(rng.integers(0, 50_000, n // 2).astype(np.int64), rng.random(n // 2) < 0.01), (np.arange(n // 2, dtype=np.int64), None)]
    for desc in (False, True):
        so, si = _sorted_by_gpu(o, [0], [desc]), _sorted_by_gpu(i, [0], [desc])
        j = api.SortMergeJoin(ctx(), N.JOIN_INNER, [N.T_INT64] * 2, [N.T_INT64] * 2, [0], [0], desc=[desc])
        j.inner_consume(si)
        j.inner_finish()
        got = j.join(so)
        j.close()
        h = api.HashJoin(ctx(), N.JOIN_INNER, [N.T_INT64] * 2, [N.T_INT64] * 2, [0], [0])
        h.build_consume(i)
        h.build_finish()
        want = h.probe(o)
        h.close()
        g = np.stack([np.asarray(c[0]) for c in got], 1)
        w = np.stack([np.asarray(c[0]) for c in want], 1)
        assert g.shape == w.shape
        assert np.array_equal(g[np.lexsort(g.T[::-1])], w[np.lexsort(w.T[::-1])])
        d = np.diff(g[:, 0])
        assert (d <= 0).all() if desc else (d >= 0).all()


def test_smj_then_sortagg_equals_join_then_hash_agg():
    rng = np.random.default_rng(11)
    ko = np.sort(rng.integers(0, 5000, 200_000)).astype(np.int64)
    ki = np.sort(rng.integers(0, 5000, 20_000)).astype(np.int64)
    o = [(ko, None), (rng.integers(-100, 100, ko.size).astype(np.int64), None)]
    i = [(ki, None), (rng.integers(-100, 100, ki.size).astype(np.int64), None)]
    j = api.SortMergeJoin(ctx(), N.JOIN_INNER, [N.T_INT64] * 2, [N.T_INT64] * 2, [0], [0])
    j.inner_consume(i)
    j.inner_finish()
    joined = j.join(o)
    j.close()
    aggs = [(N.AGG_COUNT_STAR, []), (N.AGG_SUM0, [1]), (N.AGG_SUM0, [3]), (N.AGG_MIN, [3]), (N.AGG_MAX, [1])]
    sa = api.SortAgg(ctx(), [N.T_INT64] * 4, [0], aggs)
    sa.consume(joined)
    got = sa.result()
    sa.close()
    h = api.HashJoin(ctx(), N.JOIN_INNER, [N.T_INT64] * 2, [N.T_INT64] * 2, [0], [0])
    h.build_consume(i)
    h.build_finish()
    hj = h.probe(o)
    h.close()
    ha = api.HashAgg(ctx(), [N.T_INT64] * 4, [0], aggs)
    ha.consume(hj)
    want = ha.result()
    ha.close()
    g, w = sorted(cols_to_rows(got)), sorted(cols_to_rows(want))
    assert g == w and cols_to_rows(got) == g  # the sorted aggregation keeps the join's key order


def test_operator_streams_chunks_and_closes_idempotently():
    I = ops.DataTypes.LongType
    outer = ops.MockExec([I, I], [ops.Chunk(ops.LongBlock(np.arange(k, k + 100, dtype=np.int64)), ops.LongBlock(np.zeros(100, np.int64)))
                                  for k in range(0, 1000, 100)])
    inner = ops.MockExec([I], [ops.Chunk(ops.LongBlock(np.repeat(np.arange(0, 1000, 2, dtype=np.int64), 3)))])
    ex = ops.GpuSortMergeJoinExec(outer, inner, N.JOIN_INNER, False, [ops.EquiJoinKey(0, 0, I)], [True],
                                  context=ops.ExecutionContext(chunk_size=64, gpu_batch_rows=250))
    chunks = ops.SingleExecTest(ex).exec().result()
    assert all(c.getPositionCount() <= 64 for c in chunks)
    rows = [r for c in chunks for r in c.rows()]
    assert [r[0] for r in rows] == list(np.repeat(np.arange(0, 1000, 2), 3))
    ex.close()
    ex.close()


def test_hundred_million_outer_rows():
    n = 100_000_000
    import torch
    ko = torch.arange(n, dtype=torch.int64, device="cuda") // 2
    ki = torch.arange(0, n // 2, 3, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()  # the library's stream does not wait for torch's
    j = api.SortMergeJoin(ctx(), N.JOIN_LEFT, [N.T_INT64], [N.T_INT64], [0], [0])
    try:
        j.inner_consume([(ki, None)])
        j.inner_finish()
        assert j.probe([(ko, None)]) == n
        (o, _), (k, knl) = j.next(n, N.MEM_DEVICE)
        assert j.next(1, N.MEM_DEVICE)[0][0].shape[0] == 0
    finally:
        j.close()
    assert torch.equal(o, ko)
    matched = (ko % 3) == 0
    assert torch.equal(knl.bool(), ~matched) and torch.equal(k[matched], ko[matched])
