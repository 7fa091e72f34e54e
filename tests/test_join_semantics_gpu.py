"""The GPU hash join (gsql_join_*) against the join by definition (tests/hash_join_ref.py), bit for bit.

Every case of tests/join_cases.py runs with host and device batches, through the build split into batches (a NULL
mask only on the batches that hold a NULL), probes split into batches with an empty one among them, probe_count
checked against every probe, and -- for build_outer -- unmatched_build after the last probe.  Each case whose single
key is an integer also runs with GSQL_JOIN_NO_FAST=1, and info().fast_path says which table answered.  Where the
oracle's answer does not depend on its hash layout, the GPU must equal it too.
Run on an H100 with `pytest -m gpu`.
"""
import functools

import numpy as np
import pytest

from oracle import oracle as orc
from tests import hash_join_ref as ref
from tests import join_cases as jc

pytestmark = pytest.mark.gpu

CASES = jc.cases_by_id()


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing
    return gpu_util


@functools.lru_cache(maxsize=None)
def expected(cid):
    c = CASES[cid]
    try:
        return ref.hash_join(c["spec"], c["outer"], c["inner"])
    except ref.MoreThanOneRow as e:
        return e


@functools.lru_cache(maxsize=None)
def expected_bits(cid):
    return ref.rows_bits(expected(cid))


@functools.lru_cache(maxsize=None)
def oracle_result(cid):
    c = CASES[cid]
    try:
        return orc.hash_join(c["spec"], c["outer"], c["inner"])
    except orc.MoreThanOneRow as e:
        return e


def _types(cols):
    from galaxysql_b200 import native as N
    return [{np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}[np.asarray(d).dtype]
            for d, _ in cols]


def _slice(cols, a, b, sparse_masks):
    """Rows [a, b); with sparse_masks a batch carries a column's mask only if it holds a NULL there."""
    out = []
    for d, nl in cols:
        m = None if nl is None else np.asarray(nl)[a:b].astype(np.uint8)
        if sparse_masks and m is not None and not m.any():
            m = None
        out.append((np.asarray(d)[a:b], m))
    return out


def _concat(parts, ncols):
    parts = [p for p in parts if len(p[0][0])] or parts[:1]
    return [(np.concatenate([p[c][0] for p in parts]),
             np.concatenate([np.zeros(len(p[c][0]), bool) if p[c][1] is None else p[c][1] for p in parts]))
            for c in range(ncols)]


def make_join(gu, spec, outer, inner):
    from galaxysql_b200 import api
    return api.HashJoin(gu.ctx(), spec.join_type, _types(outer), _types(inner), list(spec.outer_keys),
                        list(spec.inner_keys), list(spec.key_types), max_one_row=spec.max_one_row,
                        build_outer=spec.build_outer, anti_operands=spec.anti_operands, cond_ne=spec.cond_ne)


def probe_once(gu, j, cols, mem, capacity=None, nullable=True):
    """One gsql_join_probe into caller buffers whose masks start all-zero (a NULL the kernel fails to flag shows), with
    the E_CAPACITY retry.  -> (numpy columns, number of E_CAPACITY answers)."""
    import torch
    from galaxysql_b200 import native as N
    rows = len(cols[0][0])
    cap = max(rows, 1) if capacity is None else capacity
    retries = 0
    while True:
        out = []
        for t in j.out_types:
            dt = {N.T_INT32: np.int32, N.T_INT64: np.int64, N.T_FP64: np.float64}[t]
            d, nl = np.zeros(max(cap, 1), dt), (np.zeros(max(cap, 1), np.uint8) if nullable else None)
            if mem == "device":
                d, nl = torch.from_numpy(d).cuda(), (None if nl is None else torch.from_numpy(nl).cuda())
            out.append((d, nl))
        src = gu.to_device(cols) if mem == "device" else cols
        try:
            n = j.probe_into(src, out, cap)
        except N.CapacityError as e:
            assert e.required > cap
            cap, retries = e.required, retries + 1
            continue
        res = gu.to_numpy([(d[:n], None if nl is None else nl[:n]) for d, nl in out])
        return res, retries


def run_gpu(gu, c, mem, build_ref=False):
    """The case through the C-ABI -> (output columns, JoinInfo).  probe_count must equal every probe's row count."""
    spec, outer, inner = c["spec"], c["outer"], c["inner"]
    j = make_join(gu, spec, outer, inner)
    try:
        build, probe = (outer, inner) if spec.build_outer else (inner, outer)
        nb = len(build[0][0])
        if build_ref and mem == "device":
            j.build_consume_ref(gu.to_device(_slice(build, 0, nb, True)))
        else:
            edges = np.linspace(0, nb, c["build_parts"] + 1).astype(int)
            for a, b in zip(edges[:-1], edges[1:]):
                part = _slice(build, a, b, True)
                j.build_consume(gu.to_device(part) if mem == "device" else part)
        j.build_finish()
        info = j.info()
        npr = len(probe[0][0])
        edges = np.linspace(0, npr, c["probe_parts"] + 1).astype(int).tolist()
        if c["probe_parts"] > 1:
            edges.insert(1, edges[1])  # an empty probe batch among the others
        parts = []
        for a, b in zip(edges[:-1], edges[1:]):
            part = _slice(probe, a, b, False)
            count = j.probe_count(gu.to_device(part) if mem == "device" else part)
            got, _ = probe_once(gu, j, part, mem)
            assert count == len(got[0][0]), f"probe_count {count}, probe returned {len(got[0][0])}"
            parts.append(got)
        if spec.build_outer:
            from galaxysql_b200 import native as N
            parts.append(gu.to_numpy(j.unmatched_build(N.MEM_DEVICE if mem == "device" else N.MEM_HOST)))
        return _concat(parts, len(j.out_types)), info
    finally:
        j.close()


def fast_expected(c) -> bool:
    """Whether build_finish should pick the single-integer-key table (join.cu fast_build)."""
    spec, inner = c["spec"], c["inner"]
    if len(spec.outer_keys) != 1 or spec.build_outer or spec.max_one_row or spec.cond_ne:
        return False
    kt = spec.key_types[0]
    bk, pk = np.asarray(inner[spec.inner_keys[0]][0]), np.asarray(c["outer"][spec.outer_keys[0]][0])
    if kt == jc.F64 or bk.dtype == np.float64 or pk.dtype == np.float64:
        return False
    if kt == jc.I32 and (bk.dtype != np.int32 or pk.dtype != np.int32):
        return False
    if len(bk) == 0 or any(nl is not None and np.asarray(nl).any() for _, nl in inner):
        return False
    return len(np.unique(bk)) == len(bk) and not (bk == jc.INT64_MIN).any()  # INT64_MIN is the table's empty key


def _single_int_key(c) -> bool:
    s = c["spec"]
    return len(s.outer_keys) == 1 and s.key_types[0] in (jc.I32, jc.I64) and \
        np.asarray(c["outer"][s.outer_keys[0]][0]).dtype != np.float64 and \
        np.asarray(c["inner"][s.inner_keys[0]][0]).dtype != np.float64


PARAMS = [(cid, mem, path) for cid in CASES for mem in ("host", "device")
          for path in (("default", "generic") if _single_int_key(CASES[cid]) else ("default",))]


@pytest.mark.parametrize("cid, mem, path", PARAMS, ids=[f"{a}-{b}-{p}" for a, b, p in PARAMS])
def test_join_equals_reference(gu, monkeypatch, cid, mem, path):
    from galaxysql_b200 import native as N
    c = CASES[cid]
    if path == "generic":
        monkeypatch.setenv("GSQL_JOIN_NO_FAST", "1")
    exp = expected(cid)
    if isinstance(exp, ref.MoreThanOneRow):
        with pytest.raises(N.MoreThanOneRowError):
            run_gpu(gu, c, mem)
        if c["oracle"]:
            assert isinstance(oracle_result(cid), orc.MoreThanOneRow)
        return
    got, info = run_gpu(gu, c, mem)
    assert info.fast_path == (path == "default" and fast_expected(c)), f"fast_path={info.fast_path}"
    bits = ref.rows_bits(got)
    if bits != expected_bits(cid):
        ref.assert_rows_equal(got, exp, cid)
    if c["oracle"] and bits != ref.rows_bits(oracle_result(cid)):
        ref.assert_rows_equal(got, oracle_result(cid), f"{cid} vs oracle")
    assert [np.asarray(d).dtype for d, _ in got] == [np.asarray(d).dtype for d, _ in exp]


@pytest.mark.parametrize("cid", ["plain-inner", "notin-2col-null0", "build-outer-left", "keys3", "masks-last-of-3-left"])
def test_build_consume_ref(gu, cid):
    got, _ = run_gpu(gu, CASES[cid], "device", build_ref=True)
    ref.assert_rows_equal(got, expected(cid), cid)


# ---------------------------------------------------------------------------------------------- signed zeros
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("n_build", [100, 8192, 8193, 20000])
@pytest.mark.parametrize("nkeys", [1, 2])
def test_signed_zero_keys_match_by_bits(gu, n_build, nkeys, mem):
    """-0.0 joins only -0.0, +0.0 only +0.0, NaN nothing -- at every build size (the oracle agrees only above 8192
    build rows, where its -0.0 and +0.0 hashes stop sharing a bucket)."""
    keys = np.arange(n_build, dtype=np.float64)
    keys[1] = -0.0
    inner = [(keys, None), (np.arange(n_build, dtype=np.int32), None), (np.zeros(n_build, np.int64), None)]
    pk = jc.f64_array([jc.NEG_ZERO, jc.POS_ZERO] + jc.NANS + [jc.NEG_ZERO])
    outer = [(pk, None), (np.arange(len(pk), dtype=np.int32) + 100, None), (np.zeros(len(pk), np.int64), None)]
    sp = jc.spec(jc.LEFT, [0, 2][:nkeys], [0, 2][:nkeys], [jc.F64, jc.I64][:nkeys])
    c = jc.case("zeros", sp, outer, inner)
    got, _ = run_gpu(gu, c, mem)
    exp = ref.hash_join(sp, outer, inner)
    ref.assert_rows_equal(got, exp, f"signed zeros, {n_build} build rows")
    pairs = sorted(zip(got[1][0].tolist(), np.where(got[4][1], -1, got[4][0]).tolist()))
    assert pairs == [(100, 1), (101, 0)] + [(102 + i, -1) for i in range(len(jc.NANS))] + [(107, 1)]


# ---------------------------------------------------------------------------------------------- refusals, errors
@pytest.mark.parametrize("bad", [
    dict(join_type=orc.JOIN_SEMI, max_one_row=True), dict(join_type=orc.JOIN_ANTI, max_one_row=True),
    dict(join_type=orc.JOIN_LEFT, build_outer=True, cond_ne=((1, 3),)),
    dict(join_type=orc.JOIN_INNER, build_outer=True, cond_ne=((1, 3),)),
    dict(join_type=orc.JOIN_SEMI, build_outer=True), dict(join_type=orc.JOIN_ANTI, build_outer=True),
    dict(join_type=orc.JOIN_INNER, cond_ne=((3, 1),)),           # inner column 1 is a DOUBLE
    dict(join_type=orc.JOIN_RIGHT, cond_ne=((1, 1),)),           # RIGHT: join row = inner || outer
])
def test_create_refuses(gu, bad):
    from galaxysql_b200 import native as N
    outer = [(np.arange(4, dtype=np.int64), None), (np.arange(4, dtype=np.int32), None)]
    inner = [(np.arange(4, dtype=np.int64), None), (np.arange(4, dtype=np.float64), None)]
    spec = orc.JoinSpec(outer_keys=[0], inner_keys=[0], key_types=[orc.T_INT64], **bad)
    with pytest.raises(ref.Unsupported):
        ref.hash_join(spec, outer, inner)
    with pytest.raises(N.GsqlError) as ei:
        make_join(gu, spec, outer, inner)
    assert ei.value.status == N.E_UNSUPPORTED


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("path", ["default", "generic"])
@pytest.mark.parametrize("jt", [orc.JOIN_LEFT, orc.JOIN_RIGHT])
def test_null_into_column_without_mask_raises(gu, monkeypatch, jt, path, mem):
    from galaxysql_b200 import native as N
    if path == "generic":
        monkeypatch.setenv("GSQL_JOIN_NO_FAST", "1")
    inner = [(np.arange(1000, dtype=np.int64), None), (np.arange(1000, dtype=np.int32), None)]
    outer = [(np.arange(500, 2500, dtype=np.int64), None), (np.arange(2000, dtype=np.int32), None)]
    j = make_join(gu, jc.spec(jt, [0], [0], [jc.I64]), outer, inner)
    try:
        j.build_consume(gu.to_device(inner) if mem == "device" else inner)
        j.build_finish()
        assert j.info().fast_path == (path == "default")
        with pytest.raises(N.GsqlError) as ei:
            probe_once(gu, j, outer, mem, nullable=False)
        assert ei.value.status == N.E_INVALID
        got, _ = probe_once(gu, j, outer, mem)        # the handle is still usable
        assert len(got[0][0]) == 2000
    finally:
        j.close()


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("cid", ["plain-inner", "heavy-dups-inner", "keys2", "build0-unique-left", "single-left"])
def test_capacity_retry(gu, cid, mem):
    """An output buffer smaller than the result: E_CAPACITY with the exact size, then the full result."""
    c = CASES[cid]
    j = make_join(gu, c["spec"], c["outer"], c["inner"])
    try:
        j.build_consume(c["inner"])
        j.build_finish()
        got, retries = probe_once(gu, j, c["outer"], mem, capacity=1)
        assert retries == (1 if len(expected(cid)[0][0]) > 1 else 0)
        ref.assert_rows_equal(got, expected(cid), cid)
    finally:
        j.close()


# ---------------------------------------------------------------------------------------------- fast handle, generic batches
def _fast_tables(n_in=6000, n_out=20000, seed=900):
    inner = [(np.argsort(jc.ku.rand_u64(n_in, seed)).astype(np.int64) * 3, None), jc.rcol(n_in, seed + 1, np.int32, 50)]
    outer = [jc.rcol(n_out, seed + 2, np.int64, 3 * n_in + 99, 0.05), jc.rcol(n_out, seed + 3, np.int32, 50, 0.05),
             jc.rcol(n_out, seed + 4, np.int64, 1 << 40)]
    return outer, inner


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("mode", ["left", "right", "anti-notin", "inner-small-capacity", "semi-small-capacity"])
def test_fast_handle_answers_generic_batches(gu, mode, mem):
    """A handle whose build went to the single-key table still answers batches that table does not take -- a probe
    batch with a NULL mask, an output capacity below the probe rows -- through the generic table, built on demand."""
    outer, inner = _fast_tables()
    jt = {"left": jc.LEFT, "right": jc.RIGHT, "anti-notin": jc.ANTI, "inner-small-capacity": jc.INNER,
          "semi-small-capacity": jc.SEMI}[mode]
    sp = jc.spec(jt, [0], [0], [jc.I64], anti_operands=[0, 1] if mode == "anti-notin" else None)
    j = make_join(gu, sp, outer, inner)
    try:
        j.build_consume(gu.to_device(inner) if mem == "device" else inner)
        j.build_finish()
        assert j.info().fast_path == 1
        exp = ref.hash_join(sp, outer, inner)
        small = mode.endswith("small-capacity")
        probe = [(d, None) for d, _ in outer] if small else outer     # masks force the generic table otherwise
        if small:
            exp = ref.hash_join(sp, probe, inner)
        assert j.probe_count(gu.to_device(probe) if mem == "device" else probe) == len(exp[0][0])
        got, _ = probe_once(gu, j, probe, mem, capacity=len(probe[0][0]) // 2 if small else None)
        ref.assert_rows_equal(got, exp, mode)
        assert j.info().fast_path == 1
        # and a NULL-free batch on the same handle still goes through the fast table
        clean = [(d[:5000].copy(), None) for d, _ in outer]
        got, _ = probe_once(gu, j, clean, mem)
        ref.assert_rows_equal(got, ref.hash_join(sp, clean, inner), mode + " (mask-free batch)")
    finally:
        j.close()
