"""-m gpu: the exchange's routing and row movement against tests/exchange_ref.py, bit for bit.

* gsql_hash_rows on every seeded case (tests/exchange_cases.py), host and device batches;
* gsql_xchg_partition on every seeded case: part counts and each destination's rows (a DOUBLE by its bits, NaN payloads
  and -0.0 included), NULL masks, round-robin, and the calls it must refuse;
* gsql_xchg_push on one rank, one case per kernel variant (k_xchg_push_w for 1 to 4 NULL-free columns with the FAST and
  the generic destination, k_xchg_push for 5 columns or NULL masks, k_xchg_bcast, round-robin), with 1, 3 and 32 slabs,
  below one tile, empty, and with one CTA per slab so that every CTA walks many tiles.
"""
import numpy as np
import pytest

from tests import exchange_cases as xc
from tests import exchange_ref as xr
from tests import kat_util as ku
from tests.hash_join_ref import rows_bits

pytestmark = pytest.mark.gpu

I32, I64, F64 = xc.I32, xc.I64, xc.F64
CASES = xc.all_cases()


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()
    return gpu_util


def _types(cols):
    return [{np.dtype(np.int32): I32, np.dtype(np.int64): I64, np.dtype(np.float64): F64}[np.asarray(d).dtype] for d, _ in cols]


def _bits(a) -> np.ndarray:
    a = np.asarray(a)
    return a.view(np.int64) if a.dtype == np.float64 else a


# ------------------------------------------------------------------------------------------------ hash_rows
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("case", [c for c in CASES if c["channels"]], ids=[c["id"] for c in CASES if c["channels"]])
def test_hash_rows_match_the_reference(gu, case, mem):
    cols, ch, kt = case["cols"], case["channels"], case["key_types"]
    got = gu.ctx().hash_rows(gu.to_device(cols) if mem == "device" else cols, ch, kt)
    got = got.cpu().numpy() if hasattr(got, "cpu") else got
    assert np.array_equal(got, xr.row_hash(cols, ch, kt))


# ------------------------------------------------------------------------------------------------ partition
def _partition(gu, x, cols, mem, out_nulls):
    """gsql_xchg_partition into output columns with NULL buffers where out_nulls[c], pre-filled with 0xAB; returns
    (status, numpy columns, part counts)."""
    import ctypes as C
    from galaxysql_b200 import api
    src = gu.to_device(cols) if mem == "device" else cols
    bv = api._BatchView(src)
    out = api._alloc_out(gu.ctx(), x.types, max(bv.rows, 1), bv.mem, out_nulls)
    for d, nl in out:
        if nl is not None:
            nl.fill_(0xAB) if hasattr(nl, "fill_") else nl.fill(0xAB)
    ob, _keep = api._out_batch(out, x.types, bv.rows, bv.mem)
    counts = (C.c_int64 * x.nparts)()
    st = gu.ctx().lib.gsql_xchg_partition(x.h, bv.ref(), C.byref(ob), counts)
    gu.ctx().sync()
    return st, gu.to_numpy(api._trim(out, bv.rows)), np.array(list(counts), dtype=np.int64)


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_partition_matches_the_reference(gu, case, mem):
    from galaxysql_b200 import api, native as N
    cols, ch, kt, n = case["cols"], case["channels"], case["key_types"], case["nparts"]
    dest = xr.destinations(cols, ch, n, kt)
    x = api.Exchange(gu.ctx(), _types(cols), ch, n, key_types=kt)
    got, counts = x.partition(gu.to_device(cols) if mem == "device" else cols)
    got = gu.to_numpy(got)
    assert counts.tolist() == xr.counts(dest, n).tolist()
    assert xr.grouped_rows(got, counts) == xr.routed_rows(cols, dest)
    if len(cols[0][0]) and n in (3, 8, 10):
        # every column with a NULL buffer in the output: the columns without one in the input read back zeros
        st, got2, counts2 = _partition(gu, x, cols, mem, [True] * len(cols))
        assert st == N.OK and counts2.tolist() == counts.tolist()
        assert xr.grouped_rows(got2, counts2) == xr.routed_rows(cols, dest)
        for (d, nl), (_, src_nl) in zip(got2, cols):
            if src_nl is None:
                assert not nl.any(), "a column without NULLs came back with NULL flags"
        # a NULL-carrying input into an output without NULL buffers is refused
        if any(nl is not None and np.asarray(nl).any() for _, nl in cols):
            st, _, _ = _partition(gu, x, cols, mem, [False] * len(cols))
            assert st == N.E_INVALID
    x.close()


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("nparts", [1, 3, 8, 1000])
def test_partition_round_robin_and_refusals(gu, nparts, mem):
    from galaxysql_b200 import api, native as N
    cols = xc.table(4097, 3, 0.03)
    x = api.Exchange(gu.ctx(), _types(cols), [0], nparts, mode=N.XCHG_RANDOM)
    got, counts = x.partition(gu.to_device(cols) if mem == "device" else cols)
    dest = xr.destinations(cols, [0], nparts, mode=xr.RANDOM)
    assert counts.tolist() == xr.counts(dest, nparts).tolist()
    assert xr.grouped_rows(gu.to_numpy(got), counts) == xr.routed_rows(cols, dest)
    x.close()
    b = api.Exchange(gu.ctx(), _types(cols), [0], nparts, mode=N.XCHG_BROADCAST)
    with pytest.raises(N.GsqlError) as e:
        b.partition(gu.to_device(cols) if mem == "device" else cols)
    assert e.value.status == N.E_UNSUPPORTED
    b.close()


def test_exchange_part_count_limit(gu):
    from galaxysql_b200 import api, native as N
    x = api.Exchange(gu.ctx(), [I64], [0], xc.MAX_PARTS)
    x.close()
    with pytest.raises(N.GsqlError) as e:
        api.Exchange(gu.ctx(), [I64], [0], xc.MAX_PARTS + 1)
    assert e.value.status == N.E_INVALID


# ------------------------------------------------------------------------------------------------ push on one rank
def _push_table(n, seed, layout):
    """Columns by layout letters: k = BIGINT key (edge values), i = INT32 (negative values), d = DOUBLE (NaN payloads,
    -0.0, subnormals), p = BIGINT payload; an upper-case letter carries NULLs (30 %)."""
    t = xc.table(n, seed, 0.0)
    src = {"k": t[1][0], "i": t[3][0], "d": t[5][0], "p": t[6][0]}
    return [ku.with_nulls(src[ch.lower()], 0.3 if ch.isupper() else 0.0, seed + j) for j, ch in enumerate(layout)]


# (id, column layout, channels, key types, mode): the kernel each one reaches
PUSH_VARIANTS = [
    ("w1-fast-i64", "k", [0], [I64], "hash"),                      # k_xchg_push_w<true, 1>
    ("w2-fast-i32", "id", [0], [I32], "hash"),                     # k_xchg_push_w<true, 2>, INT32 key as INT32
    ("w3-fast-i32w", "ikd", [0], [I64], "hash"),                   # k_xchg_push_w<true, 3>, INT32 widened to INT64
    ("w4-two-channels", "kidp", [0, 1], [I64, I32], "hash"),       # k_xchg_push_w<false, 4>
    ("w2-double-key", "di", [0], [F64], "hash"),                   # k_xchg_push_w<false, 2>
    ("w2-random", "kd", [0], [I64], "random"),                     # k_xchg_push_w<false, 2>, round-robin
    ("push-nullable-key", "Kd", [0], [I64], "hash"),               # k_xchg_push<false>
    ("push-5cols", "kidpd", [0], [I64], "hash"),                   # k_xchg_push<true>
    ("push-nullable-payload", "kIDp", [0], [I64], "hash"),         # k_xchg_push<true>
    ("push-6cols-nullable-i32w", "iKDpdi", [0], [I64], "hash"),    # k_xchg_push<true>, INT32 widened
    ("bcast", "kID", [0], [I64], "broadcast"),                     # k_xchg_bcast
]
MODES = {"hash": 0, "broadcast": 1, "random": 2}


def _concat(parts, c, nulls):
    d = np.concatenate([_bits(p[c][0]) for p in parts])
    return d, (np.concatenate([p[c][1] for p in parts]) if nulls else None)


@pytest.mark.parametrize("ctas", [None, "1"], ids=["ctas-default", "ctas-1"])
@pytest.mark.parametrize("variant", PUSH_VARIANTS, ids=[v[0] for v in PUSH_VARIANTS])
def test_push_single_rank(gu, monkeypatch, variant, ctas):
    from galaxysql_b200 import api, native as N
    name, layout, ch, kt, mode = variant
    if ctas:
        monkeypatch.setenv("GSQL_XCHG_PUSH_CTAS", ctas)
    c = gu.ctx()
    nullable = [j for j, l in enumerate(layout) if l.isupper()]
    for n in (70_001, 100, 0):
        cols = _push_table(n, 11 + n, layout)
        types = _types(cols)
        cap = max(n, 1)
        x = api.Exchange(c, types, ch, 1, key_types=kt, mode=MODES[mode])
        x.open_p2p(cap, nullable=nullable)
        for nslabs in (1, 3, 32):
            slab_rows = x.push(gu.to_device(cols), nslabs)
            x.push_wait()
            whole = x.recv(-1)
            parts = [x.recv(i) for i in range(nslabs)]
            c.sync()
            whole, parts = gu.to_numpy(whole), [gu.to_numpy(p) for p in parts]
            assert sum(slab_rows) == n and [len(p[0][0]) for p in parts] == slab_rows
            if n > 4096 and nslabs == 32:
                assert slab_rows[-1] == 0, "the trailing slabs of a 32-slab push are empty"
            assert rows_bits(whole) == rows_bits(cols), f"{name}: rows differ ({nslabs} slabs)"
            for j in range(len(cols)):  # the slabs are consecutive pieces of the whole
                d, nl = _concat(parts, j, whole[j][1] is not None)
                assert np.array_equal(d, _bits(whole[j][0]))
                if nl is not None:
                    assert np.array_equal(nl, whole[j][1])
        if nullable and n:
            # the same exchange, a batch without NULL masks: the NULL bytes it receives are all zero
            x.push(gu.to_device([(d, None) for d, _ in cols]), 3)
            x.push_wait()
            again = x.recv(-1)
            c.sync()
            again = gu.to_numpy(again)
            for j in nullable:
                assert not again[j][1].any(), "a push without masks left NULL flags behind"
            assert rows_bits(again) == rows_bits([(d, None) for d, _ in cols])
        x.close()
        if n > 1 and ctas is None:  # a receive buffer of n - 1 rows is too small, on every slab count
            small = api.Exchange(c, types, ch, 1, key_types=kt, mode=MODES[mode])
            small.open_p2p(n - 1, nullable=nullable)
            with pytest.raises(N.CapacityError) as e:
                small.push(gu.to_device(cols), 3)
            assert e.value.required == n
            small.close()
