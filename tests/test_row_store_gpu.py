"""The row store (RowStore in csrc/common.cuh) through every operator that holds rows in it: the hash join's build side,
Sort / TopN, Merge and the sort-merge join's inner side.  Each case cuts its rows into many small host, device or
alternating batches (so the store grows through several capacity doublings) in which a column's NULL mask appears only
in later batches, stops after the first ones, or flags NULLs with bytes other than 1.  Results are checked against
tests/hash_join_ref.py, sort_ref.py, merge_ref.py and smj_ref.py, and every output NULL byte must be exactly 0 or 1."""
import numpy as np
import pytest

from galaxysql_b200 import api, native as N
from oracle import oracle as orc
from tests import hash_join_ref as hjr
from tests import merge_ref as mr
from tests import smj_ref as smr
from tests import sort_ref as sr

pytestmark = pytest.mark.gpu

MEMS = ["host", "device", "mixed"]
NULL_BYTES = np.array([1, 2, 7, 255], np.uint8)


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()
    return gpu_util


def _types(cols):
    return [{np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}[d.dtype] for d, _ in cols]


def _cuts(rng, n, nb):
    return np.concatenate([[0], np.sort(rng.choice(np.arange(1, n), nb - 1, replace=False)), [n]])


def batches(rng, cols, nb, masks):
    """Cuts `cols` (values, bool NULL flags) into nb batches.  Column c carries a mask in batch b per masks[c]: 'late'
    (only in the second half of the batches), 'early' (only in the first half) or 'always'.  A batch without a mask
    has its NULLs cleared; a NULL is flagged by a byte from NULL_BYTES.  -> (batches, the columns the reference sees)."""
    n = len(cols[0][0])
    cuts = _cuts(rng, n, nb)
    out, ref = [], [(d, nl.copy()) for d, nl in cols]
    for b, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
        part = []
        for c, (d, _) in enumerate(cols):
            has = masks[c] == "always" or (masks[c] == "late") == (b >= nb // 2)
            nl = ref[c][1][lo:hi]
            if not has:
                nl[:] = False
                part.append((d[lo:hi], None))
            else:
                part.append((d[lo:hi], np.where(nl, rng.choice(NULL_BYTES, hi - lo), 0).astype(np.uint8)))
        out.append(part)
    return out, ref


def feed(gu, consume, parts, mem):
    for i, p in enumerate(parts):
        consume(gu.to_device(p) if mem == "device" or (mem == "mixed" and i % 2) else p)


def table(rng, n, types, null_rate=0.1, key_range=None):
    cols = []
    for t in types:
        if t == N.T_FP64:
            d = rng.integers(-50, 50, n).astype(np.float64) / 4
        else:
            d = rng.integers(0, key_range or 1000, n).astype(np.int32 if t == N.T_INT32 else np.int64)
        cols.append((d, rng.random(n) < null_rate))
    return cols


def assert_null_bytes(cols):
    for _, nl in cols:
        if nl is not None:
            nl = nl.cpu().numpy() if hasattr(nl, "cpu") else np.asarray(nl)
            assert set(np.unique(nl).tolist()) <= {0, 1}, "an output NULL byte other than 0 or 1"


# ------------------------------------------------------------------------------------------------ hash join build side
@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("expected", [0, 1500, 100_000])
def test_join_build_store(gu, mem, expected):
    rng = np.random.default_rng(11)
    inner = table(rng, 9000, [N.T_INT64, N.T_INT32, N.T_FP64], key_range=6000)
    outer = [(rng.integers(0, 6000, 4000).astype(np.int64), None), (np.arange(4000, dtype=np.int32), None)]
    parts, ref_inner = batches(rng, inner, 37, ["late", "early", "always"])
    spec = orc.JoinSpec(orc.JOIN_LEFT, [0], [0], [orc.T_INT64])
    j = api.HashJoin(gu.ctx(), spec.join_type, _types(outer), _types(inner), [0], [0], [N.T_INT64],
                     expected_build_rows=expected)
    try:
        feed(gu, j.build_consume, parts, mem)
        j.build_finish()
        if expected > 9000:  # the build side was reserved at the hinted capacity
            assert j.info().device_bytes >= expected * (8 + 4 + 8 + 1)
        got = j.probe(gu.to_device(outer) if mem == "device" else outer)
    finally:
        j.close()
    assert_null_bytes(got)
    hjr.assert_rows_equal(gu.to_numpy(got), hjr.hash_join(spec, outer, ref_inner), f"LEFT join, {mem} build")


@pytest.mark.parametrize("mem", MEMS)
def test_join_not_in_late_null_byte(gu, mem):
    """A single build column whose only NULL (byte 255) arrives in a later batch's mask: NOT IN returns nothing."""
    rng = np.random.default_rng(12)
    d = rng.integers(0, 100, 3000).astype(np.int64)
    nl = np.zeros(3000, bool)
    nl[2500] = True
    parts = [[(d[:1000], None)], [(d[1000:2000], None)], [(d[2000:], np.where(nl[2000:], 255, 0).astype(np.uint8))]]
    outer = [(np.arange(200, 300, dtype=np.int64), None)]
    spec = orc.JoinSpec(orc.JOIN_ANTI, [0], [0], [orc.T_INT64], anti_operands=[0])
    j = api.HashJoin(gu.ctx(), spec.join_type, [N.T_INT64], [N.T_INT64], [0], [0], [N.T_INT64], anti_operands=[0])
    try:
        feed(gu, j.build_consume, parts, mem)
        j.build_finish()
        got = gu.to_numpy(j.probe(outer))
    finally:
        j.close()
    exp = hjr.hash_join(spec, outer, [(d, nl)])
    assert len(exp[0][0]) == 0
    hjr.assert_rows_equal(got, exp, f"NOT IN, {mem} build")


# ------------------------------------------------------------------------------------------------ Sort / TopN
@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("limit,nb", [(None, 41), (40_000, 6), (300, 41)])
def test_sort_store(gu, mem, limit, nb):
    """Full sort; a TopN whose batches are at most L rows (appended as they are, then cut back to L); a TopN whose
    batches exceed L (each batch's best L rows appended)."""
    rng = np.random.default_rng(13)
    n = 100_000 if limit == 40_000 else 12_000
    cols = table(rng, n, [N.T_INT32, N.T_FP64, N.T_INT64])
    parts, ref = batches(rng, cols, nb, ["late", "always", "early"])
    keys, desc = [0, 1, 2], [False, True, False]
    s = api.Sort(gu.ctx(), _types(cols), keys, desc, limit)
    try:
        feed(gu, s.consume, parts, mem)
        got = s.result(N.MEM_DEVICE if mem == "device" else N.MEM_HOST)
    finally:
        s.close()
    assert_null_bytes(got)
    sr.check_ordered(gu.to_numpy(got), ref, _types(cols), keys, desc, limit)


# ------------------------------------------------------------------------------------------------ Merge
@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("limit", [None, 2500])
def test_merge_store(gu, mem, limit):
    rng = np.random.default_rng(14)
    types = [N.T_INT64, N.T_INT32, N.T_FP64]
    keys, desc = [0], [False]
    m = api.Merge(gu.ctx(), types, keys, desc, 3, limit)
    refs = []
    try:
        for i in range(3):
            cols = table(rng, 4000 + 1000 * i, types)
            p = sr.lexsort_perm(cols, types, keys, desc)
            cols = [(d[p], nl[p]) for d, nl in cols]
            parts, ref = batches(rng, cols, 13, ["always", "late", "early"])
            refs.append(ref)
            feed(gu, lambda b, i=i: m.consume(i, b), parts, mem)
        m.finish()
        got = m.next(20_000, N.MEM_DEVICE if mem == "device" else N.MEM_HOST)
    finally:
        m.close()
    assert_null_bytes(got)
    mr.assert_rows_equal(gu.to_numpy(got), mr.merged(refs, types, keys, desc, limit))


# ------------------------------------------------------------------------------------------------ sort-merge join inner side
def _smj_rows(cols):
    rows = sr.rows_of([(d, None if nl is None else np.asarray(nl).astype(bool)) for d, nl in cols])
    return [tuple(None if v is None else (float(v) if isinstance(v, float) else int(v)) for v in r) for r in rows]


def _smj_probe(gu, ctx, inner_parts, outer, mem):
    j = api.SortMergeJoin(ctx, N.JOIN_LEFT, [N.T_INT64, N.T_INT32], [N.T_INT64, N.T_INT32, N.T_FP64], [0], [0], [N.T_INT64])
    feed(gu, j.inner_consume, inner_parts, mem)
    j.inner_finish()
    return j, j.probe(gu.to_device(outer) if mem == "device" else outer)


def _smj_drain(j, n, mem):
    got = j.next(max(n, 1), N.MEM_DEVICE if mem == "device" else N.MEM_HOST)
    assert len(got[0][0]) == n and len(j.next(1)[0][0]) == 0
    return got


def _smj_case(rng):
    types = [N.T_INT64, N.T_INT32, N.T_FP64]
    inner = table(rng, 9000, types, key_range=3000)
    p = sr.lexsort_perm(inner, types, [0], [False])
    inner = [(d[p], nl[p]) for d, nl in inner]
    parts, ref = batches(rng, inner, 37, ["always", "late", "early"])
    ok = np.sort(rng.integers(0, 3000, 2000)).astype(np.int64)
    outer = [(ok, None), (np.arange(2000, dtype=np.int32), None)]
    exp = smr.smj_ref(_smj_rows(outer), _smj_rows(ref), smr.LEFT, [0], [0], ["int"], n_inner_cols=3)
    return parts, outer, exp


@pytest.mark.parametrize("mem", MEMS)
def test_smj_inner_store(gu, mem):
    parts, outer, exp = _smj_case(np.random.default_rng(15))
    j, n = _smj_probe(gu, gu.ctx(), parts, outer, mem)
    try:
        got = _smj_drain(j, n, mem)
    finally:
        j.close()
    assert_null_bytes(got)
    assert _smj_rows(gu.to_numpy(got)) == [tuple(r) for r in exp]


def test_smj_destroyed_after_context(gu):
    """The handle holds its own reference to the context: destroying the context first leaves the handle usable until
    it is destroyed."""
    parts, outer, exp = _smj_case(np.random.default_rng(16))
    ctx = api.Context(0)
    j, n = _smj_probe(gu, ctx, parts, outer, "host")
    ctx.close()
    got = _smj_drain(j, n, "host")
    j.close()
    assert _smj_rows(gu.to_numpy(got)) == [tuple(r) for r in exp]
