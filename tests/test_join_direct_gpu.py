"""The radix join's direct table: build keys whose range fits in 2^bits <= 3 x build rows slots get slot
(key - kmin) * phi64 mod 2^bits, a collision-free slot of their own, and partitions that are the slot's top bits.
Checked against the CPU oracle, row multiset exact, for every join type, packed-row width and key type, at the mode
boundary, at the edges of the 64-bit key range, for probe keys that alias a build key's slot, and for the fallbacks
(duplicate keys, KEY_EMPTY probe keys).  The table geometry the handle reports is checked
against a numpy restatement.  Run on an H100 with `pytest -m gpu`.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import kat_util as ku
from tests.test_join_build_gpu import table_geometry
from tests.test_join_scatter_gpu import LAYOUTS, _assert_same_rows, _device_view

pytestmark = pytest.mark.gpu

ALL_JOIN_TYPES = [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT, orc.JOIN_SEMI, orc.JOIN_ANTI]
KEY_EMPTY = np.iinfo(np.int64).min
I64_MAX = np.iinfo(np.int64).max
PHI = np.uint64(0x9E3779B97F4A7C15)
PART_BYTES = 64 << 10
MAX_P = 1024


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


def _clean(monkeypatch):
    for v in ("GSQL_JOIN_PART_BYTES", "GSQL_JOIN_PART_MIN_ROWS", "GSQL_JOIN_PART_BLOCK_ROWS", "GSQL_JOIN_SUB_BATCH",
              "GSQL_JOIN_SLOTS_PER_ROW"):
        monkeypatch.delenv(v, raising=False)
    return monkeypatch


@pytest.fixture
def radix(monkeypatch):
    """Radix mode at test sizes: 64 KB partitions, every probe batch partitioned."""
    _clean(monkeypatch).setenv("GSQL_JOIN_PART_BYTES", str(PART_BYTES))
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    return monkeypatch


# ------------------------------------------------------------------------------------------------ numpy restatement
def direct_geometry(keys, nrows, W, part_bytes=None):
    """(P, nslots, bits) of fast_build()'s direct table, or None when the hash table is built.  part_bytes None: the
    default settings, under which a table of <= 64 MB is not partitioned."""
    span = int(np.max(keys)) - int(np.min(keys))
    bits = max(10, span.bit_length())
    nslots = 1 << bits
    if int(np.min(keys)) == KEY_EMPTY or nslots > max(3 * nrows, 1024):
        return None
    if part_bytes is None and nslots * W * 8 <= 64 << 20:
        return 1, nslots, bits
    spp = 1
    while spp < nslots and spp * 2 * W * 8 <= (part_bytes or 16 << 20):
        spp *= 2
    while nslots // spp > MAX_P:
        spp *= 2
    return nslots // spp, nslots, bits


def direct_slot(keys, kmin, bits):
    d = np.asarray(keys).astype(np.int64).view(np.uint64) - np.uint64(np.int64(kmin).view(np.uint64))
    with np.errstate(over="ignore"):
        return (d * PHI) & np.uint64((1 << bits) - 1)


def direct_part(keys, kmin, bits, P):
    return (direct_slot(keys, kmin, bits) >> np.uint64(bits - (P.bit_length() - 1))).astype(np.int64)


# ------------------------------------------------------------------------------------------------ tables and runs
def _pays(n, dtypes, s0):
    return [((ku.rand_u64(n, s0 + i) % np.uint64(1 << 30)).astype(t), None) for i, t in enumerate(dtypes)]


def _dense_tables(keys, probe_keys, build_pay, probe_pay, seed, probe_key_col=0):
    inner = [(keys, None)] + _pays(len(keys), build_pay, seed + 10)
    outer = _pays(len(probe_keys), probe_pay, seed + 20)
    outer.insert(probe_key_col, (probe_keys, None))
    return outer, inner


def _probe_keys(keys, n, seed, miss_share=4):
    """n probe keys drawn from the build keys; every miss_share-th one moved one past a build key."""
    pk = keys[(ku.rand_u64(n, seed) % np.uint64(len(keys))).astype(np.int64)].copy()
    miss = (ku.rand_u64(n, seed + 1) % np.uint64(miss_share)) == 0
    with np.errstate(over="ignore"):
        pk[miss] += 1
    return pk


def _join(gu, jt, outer, inner, kc=0, mem="device", build_batches=1):
    """Builds in `build_batches` batches, probes once; returns (rows, info, probe kernel names)."""
    from galaxysql_b200 import api
    ctx = gu.ctx()
    kt = orc.T_INT32 if outer[kc][0].dtype == np.int32 else orc.T_INT64
    j = api.HashJoin(ctx, jt, gu._types(outer), gu._types(inner), [kc], [0], [kt])
    try:
        edges = np.linspace(0, len(inner[0][0]), build_batches + 1).astype(int)
        for a, b in zip(edges[:-1], edges[1:]):
            part = [(d[a:b], None) for d, _ in inner]
            j.build_consume(gu.to_device(part) if mem == "device" else part)
        j.build_finish()
        info = j.info()
        ctx.profile(True)
        ctx.profile_reset()
        try:
            got = gu.to_numpy(j.probe(_device_view(outer, 0) if mem == "device" else outer))
            names = set(ctx.profile_dump())
        finally:
            ctx.profile(False)
    finally:
        j.close()
    return got, info, names


def _check(gu, jt, outer, inner, kc=0, **kw):
    got, info, names = _join(gu, jt, outer, inner, kc, **kw)
    spec = orc.JoinSpec(jt, [kc], [0], [orc.T_INT32 if outer[kc][0].dtype == np.int32 else orc.T_INT64])
    _assert_same_rows(got, orc.hash_join(spec, outer, inner))
    return info, names


def _assert_direct(info, keys, W, part_bytes=None):
    geo = direct_geometry(keys, len(keys), W, part_bytes)
    assert geo is not None
    P, nslots, _ = geo
    assert info.fast_path == 1 and info.table_slots == nslots and info.partitions == P, (info.table_slots, info.partitions, geo)


# ------------------------------------------------------------------------------------------------ mode boundary
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_ANTI])
def test_direct_mode_boundary(gu, radix, jt):
    """20 000 keys spanning [0, 32767]: 2^15 slots <= 60 000 gives the direct table (8 partitions of 4096 slots).  The
    largest key moved to 32 768 needs 2^16 > 60 000 slots: the hash table of table_geometry()."""
    n = 20_000
    keys = np.sort(np.argsort(ku.rand_u64(32_766, 5))[: n - 2] + 1).astype(np.int64)
    keys = np.concatenate([[0], keys, [32_767]]).astype(np.int64)
    keys = keys[np.argsort(ku.rand_u64(n, 6))]
    outer, inner = _dense_tables(keys, _probe_keys(keys, 60_000, 7), [np.int32, np.int32], [np.int32, np.int32], seed=8)
    info, _ = _check(gu, jt, outer, inner)
    _assert_direct(info, keys, 2, PART_BYTES)
    assert (info.table_slots, info.partitions) == (1 << 15, 8)

    keys2 = keys.copy()
    keys2[keys2 == 32_767] = 32_768
    assert direct_geometry(keys2, n, 2, PART_BYTES) is None
    outer2, inner2 = _dense_tables(keys2, _probe_keys(keys2, 60_000, 9), [np.int32, np.int32], [np.int32, np.int32], seed=8)
    info2, _ = _check(gu, jt, outer2, inner2)
    P, nslots = table_geometry(n, 2, PART_BYTES)
    assert info2.fast_path == 1 and (info2.partitions, info2.table_slots) == (P, nslots)


# ------------------------------------------------------------------------------------------------ join types x widths
@pytest.mark.parametrize("mode", ["l2", "radix"])
@pytest.mark.parametrize("key_dtype", [np.int64, np.int32], ids=["bigint_key", "int_key"])
@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("jt", ALL_JOIN_TYPES)
def test_direct_join_types_and_widths(gu, monkeypatch, jt, W, key_dtype, mode):
    """Every join type, W = 1..4 packed words, INT32 and BIGINT keys, on the unpartitioned and the radix table; the
    build side arrives in three batches."""
    _clean(monkeypatch)
    if mode == "radix":
        monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(PART_BYTES))
        monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    bp, pp = LAYOUTS[W]
    kc = 1 if pp else 0
    nb = 12_000
    keys = (np.argsort(ku.rand_u64(nb, 100 + W)) - 5_000).astype(key_dtype)  # dense, spans zero
    outer, inner = _dense_tables(keys, _probe_keys(keys, 40_000, 200 + W), bp, pp, seed=300 + 10 * W + jt, probe_key_col=kc)
    info, _ = _check(gu, jt, outer, inner, kc, build_batches=3)
    _assert_direct(info, keys, W, PART_BYTES if mode == "radix" else None)
    assert (info.partitions > 1) == (mode == "radix")


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_direct_host_and_device_batches(gu, radix, jt, mem):
    nb = 30_000
    keys = (np.argsort(ku.rand_u64(nb, 11)) - 40_000).astype(np.int64)
    outer, inner = _dense_tables(keys, _probe_keys(keys, 200_000, 12), [np.int32, np.int32], [np.int32, np.int32], seed=13)
    info, _ = _check(gu, jt, outer, inner, mem=mem)
    _assert_direct(info, keys, 2, PART_BYTES)


# ------------------------------------------------------------------------------------------------ key edges
def _edge_keys(case, n):
    base = np.argsort(ku.rand_u64(n, 21)).astype(np.int64)
    if case == "negative_kmin":
        return base - 3 * n
    if case == "next_to_int64_min":
        return base + (KEY_EMPTY + 1)
    if case == "next_to_int64_max":
        return I64_MAX - base
    raise ValueError(case)


@pytest.mark.parametrize("mode", ["l2", "radix"])
@pytest.mark.parametrize("case", ["negative_kmin", "next_to_int64_min", "next_to_int64_max"])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_SEMI, orc.JOIN_ANTI])
def test_direct_key_range_edges(gu, monkeypatch, jt, case, mode):
    """Dense keys at the ends of the 64-bit range (the probe key one past the build range wraps to the other end),
    with probe keys below kmin, above kmax, in the unused tail [kmin + range, kmin + 2^bits), and equal to a build key
    plus or minus 2^bits (the same slot, another key)."""
    _clean(monkeypatch)
    if mode == "radix":
        monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(PART_BYTES))
        monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    n = 10_000
    keys = _edge_keys(case, n)
    P, nslots, bits = direct_geometry(keys, n, 2, PART_BYTES if mode == "radix" else None)
    kmin, kmax = int(keys.min()), int(keys.max())
    with np.errstate(over="ignore"):
        extra = np.array([kmin - 1, kmin - 2, kmax + 1, kmax + 2, kmin + nslots - 1, kmin + n + 5], dtype=object)
        extra = np.array([int(x) & ((1 << 64) - 1) for x in extra], dtype=np.uint64).view(np.int64)
        alias = np.concatenate([keys[:500].view(np.uint64) + np.uint64(nslots), keys[500:1000].view(np.uint64) - np.uint64(nslots)]).view(np.int64)
    assert np.array_equal(direct_slot(alias[:500], kmin, bits), direct_slot(keys[:500], kmin, bits))
    pk = np.concatenate([_probe_keys(keys, 30_000, 22), np.repeat(extra, 50), alias])
    pk = pk[np.argsort(ku.rand_u64(len(pk), 23))]
    outer, inner = _dense_tables(keys, pk, [np.int32, np.int32], [np.int32, np.int32], seed=24)
    info, _ = _check(gu, jt, outer, inner)
    _assert_direct(info, keys, 2, PART_BYTES if mode == "radix" else None)


@pytest.mark.parametrize("jt", ALL_JOIN_TYPES)
def test_direct_int32_keys_span_zero(gu, radix, jt):
    n = 16_384
    keys = (np.argsort(ku.rand_u64(n, 31)) - n // 2).astype(np.int32)
    pk = np.concatenate([_probe_keys(keys, 40_000, 32), np.array([np.iinfo(np.int32).min, np.iinfo(np.int32).max, n, -n], np.int32)])
    outer, inner = _dense_tables(keys, pk.astype(np.int32), [np.int32], [np.int32], seed=33)
    info, _ = _check(gu, jt, outer, inner)
    _assert_direct(info, keys, 2, PART_BYTES)  # the INT payload takes a word of its own


@pytest.mark.parametrize("mode", ["l2", "radix"])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_direct_full_table(gu, monkeypatch, jt, mode):
    """2^14 keys spanning exactly 2^14 values: every slot is taken, and unmatched probe keys (outside the range, and
    aliases of build keys) must end after one read, not walk a table without an empty slot."""
    _clean(monkeypatch)
    if mode == "radix":
        monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(PART_BYTES))
        monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    n = 1 << 14
    keys = (np.argsort(ku.rand_u64(n, 41)) + 1_000).astype(np.int64)
    pk = np.concatenate([_probe_keys(keys, 30_000, 42), np.arange(-200, 1_000), keys[:3_000] + n, keys[:3_000] - n]).astype(np.int64)
    pk = pk[np.argsort(ku.rand_u64(len(pk), 43))]
    outer, inner = _dense_tables(keys, pk, [np.int64], [np.int32, np.int32], seed=44)
    info, _ = _check(gu, jt, outer, inner)
    _assert_direct(info, keys, 2, PART_BYTES if mode == "radix" else None)
    assert info.table_slots == n


# ------------------------------------------------------------------------------------------------ fallbacks
@pytest.mark.parametrize("where", ["same_batch", "other_batch"])
def test_direct_duplicate_key_falls_back(gu, radix, where):
    """A duplicate key inside a dense range (its copies in one build batch, or in different ones) disables the fast
    table; the generic path gives the oracle's rows."""
    n = 20_000
    keys = np.argsort(ku.rand_u64(n, 51)).astype(np.int64)
    dup = keys[17] if where == "same_batch" else keys[n - 3]
    keys = np.concatenate([keys[:100], [dup], keys[100:]]).astype(np.int64)
    outer, inner = _dense_tables(keys, _probe_keys(keys, 50_000, 52), [np.int32, np.int32], [np.int32, np.int32], seed=53)
    got, info, _ = _join(gu, orc.JOIN_INNER, outer, inner, build_batches=3)
    assert info.fast_path == 0
    _assert_same_rows(got, orc.hash_join(orc.JoinSpec(orc.JOIN_INNER, [0], [0], [orc.T_INT64]), outer, inner))


@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_ANTI])
def test_direct_key_empty_probe_keys_spill(gu, radix, jt):
    """KEY_EMPTY probe keys cannot take the one-pass layout (they would read as gap rows): the batch re-runs on the
    exact layout and the keys find no partner."""
    radix.setenv("GSQL_JOIN_PART_BLOCK_ROWS", "16")
    n = 30_000
    keys = np.argsort(ku.rand_u64(n, 61)).astype(np.int64)
    pk = _probe_keys(keys, 1_000_000, 62)
    pk[::10_007] = KEY_EMPTY
    outer, inner = _dense_tables(keys, pk, [np.int32, np.int32], [np.int32, np.int32], seed=63)
    info, names = _check(gu, jt, outer, inner)
    _assert_direct(info, keys, 2, PART_BYTES)
    assert "join_fast_gaps_probe" in names and "join_fast_hist_probe" in names, sorted(names)


# ------------------------------------------------------------------------------------------------ one-pass regions
def _region_keys(case, n):
    if case == "dense":
        return np.argsort(ku.rand_u64(n, 81)).astype(np.int64)
    if case == "stride32":  # 8 of every 32 values, like TPC-H order keys
        i = np.argsort(ku.rand_u64(n, 82)).astype(np.int64)
        return (i // 8) * 32 + i % 8
    if case == "clustered":  # runs of 1000 keys, 100 000 apart
        i = np.argsort(ku.rand_u64(n, 83)).astype(np.int64)
        return (i // 1000) * 100_000 + i % 1000
    raise ValueError(case)


@pytest.mark.parametrize("case", ["dense", "stride32", "clustered"])
def test_direct_onepass_regions(gu, radix, case):
    """Dense, stride-32 and clustered build keys, 1 M probe rows drawn from them: the partitions are even, so the probe
    takes the one-pass layout (no probe histogram).  Each table is cut into 8 partitions."""
    radix.setenv("GSQL_JOIN_PART_BLOCK_ROWS", "16")
    radix.setenv("GSQL_JOIN_SLOTS_PER_ROW", "200")  # lets the sparser key sets take the direct table at test size
    n = 20_000
    keys = _region_keys(case, n)
    nslots = 1 << max(10, (int(keys.max()) - int(keys.min())).bit_length())
    radix.setenv("GSQL_JOIN_PART_BYTES", str(nslots * 16 // 8))
    outer, inner = _dense_tables(keys, _probe_keys(keys, 1_000_000, 84), [np.int32, np.int32], [np.int32, np.int32], seed=85)
    info, names = _check(gu, orc.JOIN_INNER, outer, inner)
    assert info.fast_path == 1 and info.table_slots == nslots and info.partitions == 8
    assert "join_fast_gaps_probe" in names and "join_fast_hist_probe" not in names, sorted(names)


def test_direct_skewed_probe_spills(gu, radix):
    """A probe side concentrated in one direct partition (found with the numpy restatement) overflows its region: the
    batch is joined again on the exact layout."""
    radix.setenv("GSQL_JOIN_PART_BLOCK_ROWS", "16")
    n = 30_000
    keys = np.argsort(ku.rand_u64(n, 91)).astype(np.int64)
    P, nslots, bits = direct_geometry(keys, n, 2, PART_BYTES)
    assert P > 2
    hot = keys[direct_part(keys, int(keys.min()), bits, P) == 1]
    pk = np.concatenate([_probe_keys(keys, 500_000, 92), _probe_keys(hot, 500_000, 93)])
    pk = pk[np.argsort(ku.rand_u64(len(pk), 94))]
    outer, inner = _dense_tables(keys, pk, [np.int32, np.int32], [np.int32, np.int32], seed=95)
    info, names = _check(gu, orc.JOIN_LEFT, outer, inner)
    _assert_direct(info, keys, 2, PART_BYTES)
    assert "join_fast_gaps_probe" in names and "join_fast_hist_probe" in names, sorted(names)
