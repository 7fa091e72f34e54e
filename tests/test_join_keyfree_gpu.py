"""The direct join table stores no keys: (W - 1) payload words per slot plus an occupancy bitmap, and a probe key k
matches when k - kmin is below 2^bits and its slot's bit is set.  Every case is held against the join by definition
(tests/hash_join_ref.py), on the unpartitioned (P == 1) table and on the radix table (forced with
GSQL_JOIN_PART_BYTES): key-only build sides (bitmap alone), probe keys that alias a build key's slot from outside the
range (for build keys that are a whole range of values, which the probe tests without the bitmap, and for keys with
gaps), build keys starting at the BIGINT minimum (no reserved key), duplicate build keys (the generic path takes
over), NULL padding of LEFT and RIGHT joins, slot blocks larger than the table and blocks so small that build rows
leave their split CTA's window.  The table size the handle reports is checked against the layout.
Run on an H100 with `pytest -m gpu`.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import hash_join_ref as ref
from tests import kat_util as ku
from tests.test_join_direct_gpu import PART_BYTES, _clean, _dense_tables, _join, _probe_keys, direct_slot
from tests.test_join_scatter_gpu import LAYOUTS

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


def _mode(monkeypatch, mode):
    _clean(monkeypatch)
    monkeypatch.delenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", raising=False)
    if mode == "radix":
        monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(PART_BYTES))
        monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    return PART_BYTES if mode == "radix" else None


def _check(gu, jt, outer, inner, kc=0, **kw):
    got, info, names = _join(gu, jt, outer, inner, kc, **kw)
    kt = ref.T_INT32 if outer[kc][0].dtype == np.int32 else ref.T_INT64
    ref.assert_rows_equal(got, ref.hash_join(orc.JoinSpec(jt, [kc], [0], [kt]), outer, inner), f"join type {jt}")
    return info, names


def _geometry(keys, W, part_bytes):
    """(P, nslots) of the direct table for keys whose range fits it: partitions of the slots that W * 8-byte slots of
    part_bytes give (part_bytes None: the unpartitioned table of a test-sized build)."""
    nslots = 1 << max(10, (int(np.max(keys)) - int(np.min(keys))).bit_length())
    if part_bytes is None:
        return 1, nslots
    spp = 1
    while spp < nslots and spp * 2 * W * 8 <= part_bytes:
        spp *= 2
    while nslots // spp > 1024:
        spp *= 2
    return nslots // spp, nslots


def _assert_keyfree(info, keys, W, part_bytes):
    """The direct table, (W - 1) * 8 bytes and one bit per slot."""
    P, nslots = _geometry(keys, W, part_bytes)
    assert info.fast_path == 1 and (info.partitions, info.table_slots) == (P, nslots), (info.fast_path, info.partitions, info.table_slots, P, nslots)
    assert info.table_bytes == nslots * (W - 1) * 8 + nslots // 8, (info.table_bytes, nslots, W)


# ------------------------------------------------------------------------------------------------ key-only build side
@pytest.mark.parametrize("mode", ["l2", "radix"])
@pytest.mark.parametrize("key_dtype", [np.int64, np.int32], ids=["bigint_key", "int_key"])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_SEMI, orc.JOIN_ANTI])
def test_keyfree_key_only_build(gu, monkeypatch, jt, key_dtype, mode):
    """A build side of the key alone: the table is the bitmap, nslots / 8 bytes."""
    part_bytes = _mode(monkeypatch, mode)
    n = 50_000
    keys = (np.argsort(ku.rand_u64(n, 501)) * 2 - 30_000).astype(key_dtype)  # every other value: half the slots taken
    pk = _probe_keys(keys, 120_000, 502, miss_share=3)
    outer, inner = _dense_tables(keys, pk.astype(key_dtype), [], [np.int32, np.int64], seed=503)
    info, _ = _check(gu, jt, outer, inner, build_batches=2)
    _assert_keyfree(info, keys, 1, part_bytes)


# ------------------------------------------------------------------------------------------------ aliasing probe keys
@pytest.mark.parametrize("fill", ["dense", "gaps"])
@pytest.mark.parametrize("mode", ["l2", "radix"])
@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT, orc.JOIN_SEMI, orc.JOIN_ANTI])
def test_keyfree_aliasing_probe_keys(gu, monkeypatch, jt, W, mode, fill):
    """Probe keys k + j * 2^bits (j = +-1, +-2, and 2^63 / 2^bits: the same slot as a build key, another key), keys
    below kmin, in the unused tail of the slot range, and the BIGINT extremes: the range test rejects them all, whatever
    the bit of the slot they alias says.  LEFT and RIGHT pad them with NULLs.  Build keys that are a whole range
    (dense: the range test alone decides) or a third of the values missing from it (the bitmap decides)."""
    part_bytes = _mode(monkeypatch, mode)
    bp, pp = LAYOUTS[W]
    kc = 1 if pp else 0
    n = 12_000
    keys = np.argsort(ku.rand_u64(n, 510 + W)).astype(np.int64)
    if fill == "gaps":
        keys = keys * 3 // 2
    keys = keys + 1_000_000
    kmin = int(keys.min())
    nslots = 1 << max(10, (int(keys.max()) - kmin).bit_length())
    bits = nslots.bit_length() - 1
    sel = keys[:400].view(np.uint64)
    with np.errstate(over="ignore"):
        alias = np.concatenate([sel + np.uint64(j * nslots & (2**64 - 1)) for j in (1, -1, 2, -2)]
                               + [sel + np.uint64(1 << 63)]).view(np.int64)
    assert np.array_equal(direct_slot(alias[:400], kmin, bits), direct_slot(keys[:400], kmin, bits))
    extra = np.array([I64_MIN, I64_MIN + 1, I64_MAX, I64_MAX - 1, kmin - 1, kmin - nslots, 0, -1, kmin + n, kmin + nslots - 1], np.int64)
    pk = np.concatenate([_probe_keys(keys, 30_000, 520 + W), alias, np.repeat(extra, 20)])
    pk = pk[np.argsort(ku.rand_u64(len(pk), 530 + W))]
    outer, inner = _dense_tables(keys, pk, bp, pp, seed=540 + W, probe_key_col=kc)
    info, _ = _check(gu, jt, outer, inner, kc)
    _assert_keyfree(info, keys, W, part_bytes)


# ------------------------------------------------------------------------------------------------ no reserved key
@pytest.mark.parametrize("mode", ["l2", "radix"])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_keyfree_build_keys_from_int64_min(gu, monkeypatch, jt, mode):
    """Build keys [INT64_MIN, INT64_MIN + n): the hash table's empty marker is an ordinary key of the direct table.
    Probe keys equal to it match; in radix mode they make the one-pass probe layout re-run on the exact one."""
    part_bytes = _mode(monkeypatch, mode)
    n = 20_000
    keys = (np.argsort(ku.rand_u64(n, 551)).astype(np.int64) + I64_MIN).astype(np.int64)
    pk = np.concatenate([_probe_keys(keys, 60_000, 552), np.full(37, I64_MIN, np.int64), np.array([I64_MAX, I64_MIN + n], np.int64)])
    pk = pk[np.argsort(ku.rand_u64(len(pk), 553))]
    outer, inner = _dense_tables(keys, pk, [np.int32, np.int32], [np.int32, np.int32], seed=554)
    info, _ = _check(gu, jt, outer, inner, build_batches=2)
    _assert_keyfree(info, keys, 2, part_bytes)


# ------------------------------------------------------------------------------------------------ duplicates
@pytest.mark.parametrize("blocks", ["default", "tiny"])
@pytest.mark.parametrize("mode", ["l2", "radix"])
@pytest.mark.parametrize("W", [1, 2])
def test_keyfree_duplicate_keys_fall_back(gu, monkeypatch, W, mode, blocks):
    """A duplicated build key (inside the range, across build batches) is found by its slot's bit being set already;
    the generic path answers.  Tiny slot blocks also send build rows past their split CTA's window to the deferred
    insert, which finds the duplicates there."""
    _mode(monkeypatch, mode)
    stride = 1
    if blocks == "tiny":  # keys 32 apart in 32-slot blocks (see test_keyfree_slot_blocks)
        monkeypatch.setenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", "32")
        monkeypatch.setenv("GSQL_JOIN_SLOTS_PER_ROW", "64")
        stride = 32
    bp, pp = LAYOUTS[W]
    n = 20_000
    keys = np.argsort(ku.rand_u64(n, 561)).astype(np.int64) * stride
    keys = np.concatenate([keys[:50], keys[[7, n - 1, 12_345]], keys[50:]]).astype(np.int64)
    outer, inner = _dense_tables(keys, _probe_keys(keys, 50_000, 562), bp, pp, seed=563, probe_key_col=1 if pp else 0)
    got, info, _ = _join(gu, orc.JOIN_INNER, outer, inner, 1 if pp else 0, build_batches=3)
    assert info.fast_path == 0
    ref.assert_rows_equal(got, ref.hash_join(orc.JoinSpec(orc.JOIN_INNER, [1 if pp else 0], [0], [ref.T_INT64]), outer, inner))


# ------------------------------------------------------------------------------------------------ slot blocks
@pytest.mark.parametrize("block_slots", ["32", "default"])
@pytest.mark.parametrize("W", [1, 2, 4])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_SEMI])
def test_keyfree_slot_blocks(gu, monkeypatch, jt, W, block_slots):
    """Radix builds.  Keys 32 apart (GSQL_JOIN_SLOTS_PER_ROW lets them take the direct table): with 32-slot blocks a
    split CTA's rows span more blocks than its window, and the rows beyond it go to k_fj_insert<W, true>.  Then a
    1024-slot table in 4 KB partitions, smaller than one default block (a single ragged block)."""
    _mode(monkeypatch, "radix")
    monkeypatch.setenv("GSQL_JOIN_SLOTS_PER_ROW", "64")
    if block_slots != "default":
        monkeypatch.setenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", block_slots)
    bp, pp = LAYOUTS[W]
    kc = 1 if pp else 0
    for n, stride, part_bytes, seed in ((20_000, 32, PART_BYTES, 571), (700, 1, 4096, 572)):
        monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(part_bytes))
        keys = (np.argsort(ku.rand_u64(n, seed)) * stride - 77).astype(np.int64)
        outer, inner = _dense_tables(keys, _probe_keys(keys, 3 * n, seed + 10), bp, pp, seed=seed + 20, probe_key_col=kc)
        info, _ = _check(gu, jt, outer, inner, kc)
        _assert_keyfree(info, keys, W, part_bytes)
