"""-m gpu checks of how every operator that returns rows writes its `out` batch, in both memory spaces: a device batch is
written in place, a host batch through device scratch columns and one download.  Each entry point is run once with the
NULL buffers its rule asks for (the rows and their NULLs must come back) and once without them (GSQL_E_INVALID), on the
same handle, so the refusal is also seen to leave the handle usable.  The rules (include/gsql_gpu.h):
  (a) a NULL must not be written into a column without a nulls buffer: join probe / unmatched build, scan, bloom filter,
      sort, merge, sort-merge join;
  (b) every out column needs a nulls buffer: hash aggregation, grouping sets, sorted aggregation, window, wire decoder;
  (c) exchange partition: an out column needs a nulls buffer where the input column has one."""
import ctypes as C

import numpy as np
import pytest

from galaxysql_b200 import api, native as N

pytestmark = pytest.mark.gpu

MEMS = [N.MEM_HOST, N.MEM_DEVICE]


@pytest.fixture(scope="module")
def ctx():
    from tests import gpu_util
    return gpu_util.ctx()


def _in(cols, mem):
    """numpy (values, nulls) columns, uploaded for a device batch."""
    from tests import gpu_util
    cols = [(np.asarray(d), None if nl is None else np.asarray(nl, dtype=bool)) for d, nl in cols]
    return gpu_util.to_device(cols) if mem == N.MEM_DEVICE else cols


def _np(cols):
    from tests import gpu_util
    return [(d, np.zeros(len(d), bool) if nl is None else nl) for d, nl in gpu_util.to_numpy(cols)]


def _refused(ctx, st):
    with pytest.raises(N.GsqlError) as e:
        ctx.check(st)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value), str(e.value)


def _raw_next(ctx, fn, h, types, mem, with_nulls, max_rows):
    """One `*_next(h, out, max_rows, &n)` call into out columns with NULL buffers only where `with_nulls` says."""
    out = api._alloc_out(ctx, types, max_rows, mem, with_nulls)
    ob, _keep = api._out_batch(out, types, 0, mem)
    n = C.c_int64()
    return fn(h, C.byref(ob), max_rows, C.byref(n))


# rows already ordered on column 0 (NULLs first), with two NULL keys
SORTED = [(np.array([0, 0, 2, 3, 5], np.int64), [1, 1, 0, 0, 0]), (np.arange(5, dtype=np.int32), None)]


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_sort_next(ctx, mem):
    s = api.Sort(ctx, [N.T_INT64, N.T_INT32], [0])
    s.consume(_in(SORTED, mem))
    assert s.finish() == 5
    with pytest.raises(N.GsqlError) as e:
        s.next(5, mem, nullable_out=False)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (k, kn), (v, _) = _np(s.next(5, mem))
    assert kn.tolist() == [1, 1, 0, 0, 0] and k[2:].tolist() == [2, 3, 5] and sorted(v.tolist()) == list(range(5))
    s.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_merge_next(ctx, mem):
    m = api.Merge(ctx, [N.T_INT64, N.T_INT32], [0], [False], 1)
    m.consume(0, _in(SORTED, mem))
    assert m.finish() == 5
    with pytest.raises(N.GsqlError) as e:
        m.next(5, mem, nullable_out=False)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (k, kn), (v, _) = _np(m.next(5, mem))
    assert kn.tolist() == [1, 1, 0, 0, 0] and k[2:].tolist() == [2, 3, 5] and v.tolist() == list(range(5))
    m.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_smj_next(ctx, mem):
    j = api.SortMergeJoin(ctx, N.JOIN_INNER, [N.T_INT64, N.T_INT32], [N.T_INT64], [0], [0])
    j.inner_consume(_in([(np.array([1, 2, 3], np.int64), None)], mem))
    j.inner_finish()
    assert j.probe(_in([(np.array([1, 2, 3], np.int64), None), (np.array([10, 20, 30], np.int32), [0, 1, 0])], mem)) == 3
    with pytest.raises(N.GsqlError) as e:
        j.next(3, mem, nullable_out=False)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (ok, _), (p, pn), (ik, _) = _np(j.next(3, mem))
    assert ok.tolist() == ik.tolist() == [1, 2, 3] and pn.tolist() == [0, 1, 0] and p[pn == 0].tolist() == [10, 30]
    assert len(j.next(3, mem)[0][0]) == 0
    j.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_scan_apply(ctx, mem):
    s = api.Scan(ctx, [N.T_INT64, N.T_INT32], [api.E.col(1), api.E.col(0)], filter=api.E.col(0) > 1)
    cols = _in([(np.array([1, 2, 3, 4], np.int64), None), (np.array([5, 6, 7, 8], np.int32), [0, 0, 1, 0])], mem)
    with pytest.raises(N.GsqlError) as e:
        s.apply(cols, nullable_out=False)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (v, vn), (k, _) = _np(s.apply(cols))
    assert k.tolist() == [2, 3, 4] and vn.tolist() == [0, 1, 0] and v[vn == 0].tolist() == [6, 8]
    s.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_bloom_filter(ctx, mem):
    b = api.BloomFilter(ctx, 64 * 16, 3)
    b.put(_in([(np.array([1, 2, 3], np.int64), None)], mem))
    cols = _in([(np.array([1, 2, 3], np.int64), None), (np.array([10, 20, 30], np.int32), [0, 1, 0])], mem)
    with pytest.raises(N.GsqlError) as e:
        b.filter(cols, 0, nullable_out=False)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (k, _), (p, pn) = _np(b.filter(cols, 0))
    assert k.tolist() == [1, 2, 3] and pn.tolist() == [0, 1, 0] and p[pn == 0].tolist() == [10, 30]
    b.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_xchg_partition(ctx, mem):
    types = [N.T_INT64, N.T_INT32]
    x = api.Exchange(ctx, types, [0], 4)
    src = [(np.arange(64, dtype=np.int64), None), (np.arange(64, dtype=np.int32), np.arange(64) % 3 == 0)]
    cols = _in(src, mem)
    bv = api._BatchView(cols)
    out = api._alloc_out(ctx, types, 64, mem, [True, False])
    ob, _keep = api._out_batch(out, types, 64, mem)
    counts = (C.c_int64 * 4)()
    _refused(ctx, ctx.lib.gsql_xchg_partition(x.h, bv.ref(), C.byref(ob), counts))
    got, counts = x.partition(cols)
    (k, _), (v, vn) = _np(got)
    assert counts.sum() == 64 and sorted(k.tolist()) == list(range(64))
    assert (vn == (k % 3 == 0)).all() and (v[~vn] == k[~vn]).all()
    x.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_serde_deserialize(ctx, mem):
    types = [N.T_INT64, N.T_INT32]
    src = [(np.arange(10, dtype=np.int64), None), (np.arange(10, dtype=np.int32), np.arange(10) % 4 == 1)]
    wire = api.serde_serialize(ctx, _in(src, mem), 4)
    ptr, nbytes = (wire.data_ptr(), wire.numel()) if mem == N.MEM_DEVICE else (wire.ctypes.data, wire.size)
    out = api._alloc_out(ctx, types, 10, mem, [True, False])
    ob, _keep = api._out_batch(out, types, 0, mem)
    n = C.c_int64()
    _refused(ctx, ctx.lib.gsql_serde_deserialize(ctx.ptr, C.c_void_p(ptr), nbytes, mem, C.byref(ob), 10, C.byref(n)))
    (k, kn), (v, vn) = _np(api.serde_deserialize(ctx, wire, types))
    assert k.tolist() == list(range(10)) and not kn.any()
    assert vn.tolist() == (np.arange(10) % 4 == 1).tolist() and (v[~vn] == k[~vn]).all()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_window_apply(ctx, mem):
    w = api.Window(ctx, [N.T_INT64], [0], [(N.AGG_ROW_NUMBER, []), (N.AGG_MAX, [0])])
    cols = _in([(np.array([1, 1, 2, 2, 2], np.int64), None)], mem)
    bad = api._alloc_out(ctx, w.out_types, 5, mem, [True, False])
    with pytest.raises(N.GsqlError) as e:
        w.apply(cols, out_cols=bad)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (rn, rnn), (mx, mxn) = _np(w.apply(cols))
    assert rn.tolist() == [1, 2, 1, 2, 3] and mx.tolist() == [1, 1, 2, 2, 2] and not rnn.any() and not mxn.any()
    w.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_join_probe(ctx, mem):
    """A probe column with a NULL keeps the probe on the generic (count, scan, write) path."""
    j = api.HashJoin(ctx, N.JOIN_INNER, [N.T_INT64, N.T_INT32], [N.T_INT64], [0], [0])
    j.build_consume([(np.array([1, 2, 3, 4], np.int64), None)])
    j.build_finish()
    cols = _in([(np.array([1, 2, 3, 9], np.int64), None), (np.array([10, 20, 30, 40], np.int32), [0, 1, 0, 0])], mem)
    with pytest.raises(N.GsqlError) as e:
        j.probe(cols, capacity=4, nullable_out=False)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (ok, _), (p, pn), (ik, _) = _np(j.probe(cols, capacity=4))
    order = np.argsort(ok)
    assert ok[order].tolist() == ik[order].tolist() == [1, 2, 3] and pn[order].tolist() == [0, 1, 0]
    assert p[order][[0, 2]].tolist() == [10, 30]
    j.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_join_unmatched_build(ctx, mem):
    """LEFT join that builds its outer side: the outer rows no probe row matched come back with a NULL inner column."""
    j = api.HashJoin(ctx, N.JOIN_LEFT, [N.T_INT64], [N.T_INT64], [0], [0], build_outer=True)
    j.build_consume([(np.array([1, 2, 3], np.int64), None)])
    j.build_finish()
    assert len(j.probe([(np.array([2], np.int64), None)])[0][0]) == 1
    _refused(ctx, _raw_next(ctx, ctx.lib.gsql_join_unmatched_build, j.h, j.out_types, mem, [True, False], 4))
    (ok, _), (ik, ikn) = _np(j.unmatched_build(mem))
    assert sorted(ok.tolist()) == [1, 3] and ikn.tolist() == [1, 1]
    j.close()


GROUP_IN = [(np.array([1, 2, 1, 3, 1], np.int64), None)]


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_agg_next(ctx, mem):
    a = api.HashAgg(ctx, [N.T_INT64], [0], [(N.AGG_COUNT_STAR, [])])
    a.consume(GROUP_IN)
    assert a.finish() == 3
    _refused(ctx, _raw_next(ctx, ctx.lib.gsql_agg_next, a.h, a.out_types, mem, [False, True], 3))
    (k, kn), (c, cn) = _np(a.next(3, mem))
    assert dict(zip(k.tolist(), c.tolist())) == {1: 3, 2: 1, 3: 1} and not kn.any() and not cn.any()
    a.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_sortagg_next(ctx, mem):
    s = api.SortAgg(ctx, [N.T_INT64], [0], [(N.AGG_COUNT_STAR, [])])
    s.consume([(np.array([1, 1, 1, 2, 3], np.int64), None)])
    assert s.finish() == 3
    with pytest.raises(N.GsqlError) as e:
        s.next(3, mem, nullable_out=False)
    assert e.value.status == N.E_INVALID and "nulls buffer" in str(e.value)
    (k, kn), (c, cn) = _np(s.next(3, mem))
    assert k.tolist() == [1, 2, 3] and c.tolist() == [3, 1, 1] and not kn.any() and not cn.any()
    s.close()


@pytest.mark.parametrize("mem", MEMS, ids=["host", "device"])
def test_gsagg_next(ctx, mem):
    """GROUP BY ROLLUP(k) with its grouping id g: the grand-total set's k is a NULL constant and each set's g a constant, both
    filled in the out batch's own memory space."""
    g = api.GroupingSetsAgg(ctx, [N.T_INT64], [N.T_INT64, N.T_INT64], [[0, ("const", 0)], [None, ("const", 1)]], [0, 1],
                            [(N.AGG_COUNT_STAR, [])])
    g.consume(GROUP_IN)
    assert g.finish() == 4
    _refused(ctx, _raw_next(ctx, ctx.lib.gsql_gsagg_next, g.h, g.out_types, mem, [False, True, True], 4))
    (k, kn), (gid, gn), (c, cn) = _np(g.next(4, mem))
    assert kn.tolist() == [0, 0, 0, 1] and gid.tolist() == [0, 0, 0, 1] and not gn.any() and not cn.any()
    assert dict(zip(k[:3].tolist(), c[:3].tolist())) == {1: 3, 2: 1, 3: 1} and c[3] == 5
    g.close()
