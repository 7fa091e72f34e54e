"""The radix join's table build: rows split by slot block (k_fj_build_split), each block built in shared memory and
written whole (k_fj_build_slab), and the rows whose probe sequence leaves their block inserted afterwards into the
finished table (k_fj_insert).  Checked against the CPU oracle, row multiset exact, for every join type, packed-row
width and key type, with partitions smaller than a block, forced tiny blocks, and build keys crafted so that most
rows leave their block.  Run on an H100 with `pytest -m gpu`.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import kat_util as ku
from tests.test_join_scatter_gpu import LAYOUTS, _assert_same_rows, _check, _tables

pytestmark = pytest.mark.gpu

ALL_JOIN_TYPES = [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT, orc.JOIN_SEMI, orc.JOIN_ANTI]
KEY_EMPTY = -2**63  # the table's empty-slot marker


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


@pytest.fixture
def radix(monkeypatch):
    """Radix-partitioned path at test sizes, default build."""
    monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(64 << 10))
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    monkeypatch.delenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", raising=False)
    return monkeypatch


# ------------------------------------------------------------------------------------------------ numpy restatement
PHI = np.uint64(0x9E3779B97F4A7C15)
M32 = np.uint64(0xFFFFFFFF)


def key_hash(keys):
    """join_fast.cuh key_hash on sign-extended 64-bit keys (uint64 arithmetic wraps like the device's)."""
    k = np.asarray(keys).astype(np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        return (k ^ (k >> np.uint64(32))) * PHI


def mulhi(a, b):
    """High 64 bits of the 128-bit product of uint64 arrays a and scalar b (exact, from 32-bit halves)."""
    b = np.uint64(b)
    a_lo, a_hi, b_lo, b_hi = a & M32, a >> np.uint64(32), b & M32, b >> np.uint64(32)
    ll, hl, lh, hh = a_lo * b_lo, a_hi * b_lo, a_lo * b_hi, a_hi * b_hi
    cross = (ll >> np.uint64(32)) + (hl & M32) + lh
    return hh + (hl >> np.uint64(32)) + (cross >> np.uint64(32))


def table_geometry(build_rows, W, part_bytes):
    """(P, nslots) of fast_build() for a radix table: 3 slots per row, partitions of part_bytes."""
    want = max(build_rows * 3, 1024)
    P = min(max(-(-want * W * 8 // part_bytes), 1), 1024)
    spp = -(-want // P)
    return P, spp * P


def home_slots(keys, nslots):
    return mulhi(key_hash(keys), nslots)


def _crafted_keys(nb, block, W, part_bytes, seed):
    """nb distinct BIGINT keys whose home slot is the LAST slot of a block of `block` slots: in every block the first
    row takes that slot and every other one runs off the block's end.  Returns (keys, rows that must leave their block)."""
    _, nslots = table_geometry(nb, W, part_bytes)
    cand = np.unique((ku.rand_u64(nb * block * 3, seed) >> np.uint64(2)).astype(np.int64) - (1 << 61))
    s = home_slots(cand, nslots)
    keys = cand[(s % np.uint64(block)) == np.uint64(block - 1)][:nb]
    assert len(keys) == nb
    per_block = np.bincount((home_slots(keys, nslots) // np.uint64(block)).astype(np.int64))
    return keys, int(np.maximum(per_block - 1, 0).sum())


def _crafted_tables(keys, npr, seed):
    inner = [(keys, None), ((ku.rand_u64(len(keys), seed + 1) % np.uint64(1 << 30)).astype(np.int32), None)]
    pk = keys[(ku.rand_u64(npr, seed + 2) % np.uint64(len(keys))).astype(np.int64)].copy()
    pk[::4] += 1  # a quarter of the probe keys shifted off their build key: most of them find no partner
    outer = [(pk, None), ((ku.rand_u64(npr, seed + 3) % np.uint64(1 << 30)).astype(np.int32), None)]
    return outer, inner


def _join(gu, jt, outer, inner, launches=None):
    """Builds and probes one join; `launches`, a dict, receives the named kernel launches of the build."""
    from galaxysql_b200 import api
    ctx = gu.ctx()
    j = api.HashJoin(ctx, jt, gu._types(outer), gu._types(inner), [0], [0], [orc.T_INT64])
    try:
        j.build_consume(gu.to_device(inner))
        if launches is not None:
            ctx.profile(True)
            ctx.profile_reset()
        try:
            j.build_finish()
        finally:
            if launches is not None:
                launches.update(ctx.profile_dump())
                ctx.profile(False)
        info = j.info()
        got = gu.to_numpy(j.probe(gu.to_device(outer)))
    finally:
        j.close()
    return got, info


# ------------------------------------------------------------------------------------------------ join types x widths
@pytest.mark.parametrize("block", [None, "64"], ids=["default_block", "block64"])
@pytest.mark.parametrize("key_dtype", [np.int64, np.int32], ids=["bigint_key", "int_key"])
@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("jt", ALL_JOIN_TYPES)
def test_build_join_types_and_widths(gu, radix, jt, W, key_dtype, block):
    """Every join type on the radix path with W = 1..4 packed words and INT32 / BIGINT keys.  With the default block
    (>= 4096 slots) every block straddles several 64 KB partitions; with 64-slot blocks each partition spans many blocks."""
    if block:
        radix.setenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", block)
    bp, pp = LAYOUTS[W]
    kc = 1 if pp else 0
    outer, inner = _tables(30_000, 70_000, key_dtype, bp, pp, seed=700 + 10 * W + jt, probe_key_col=kc)
    _check(gu, jt, outer, inner, kc)


@pytest.mark.parametrize("block", [None, "16"], ids=["default_block", "block16"])
@pytest.mark.parametrize("jt", ALL_JOIN_TYPES)
def test_build_partitions_smaller_than_a_block(gu, radix, jt, block):
    """GSQL_JOIN_PART_BYTES = 4096: 72 partitions of 256 slots, far smaller than a default block; several build
    batches are concatenated before the build."""
    radix.setenv("GSQL_JOIN_PART_BYTES", "4096")
    if block:
        radix.setenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", block)
    outer, inner = _tables(6144, 20_000, np.int64, [np.int32, np.int32], [np.int32, np.int32], seed=40 + jt)
    spec = orc.JoinSpec(jt, [0], [0], [orc.T_INT64])
    got = gu.gpu_hash_join(spec, outer, inner, mem="device", build_batches=3)
    _assert_same_rows(got, orc.hash_join(spec, outer, inner))


def test_build_unpartitioned_table_untouched(gu, monkeypatch):
    """A table that fits L2 (P = 1) is still built by k_fj_table_init + k_fj_insert, never by the block build."""
    for v in ("GSQL_JOIN_PART_BYTES", "GSQL_JOIN_BUILD_BLOCK_SLOTS"):
        monkeypatch.delenv(v, raising=False)
    outer, inner = _tables(20_000, 50_000, np.int64, [np.int32, np.int32], [np.int32, np.int32], seed=9)
    launches = {}
    got, info = _join(gu, orc.JOIN_INNER, outer, inner, launches)
    assert info.fast_path == 1 and info.partitions == 1
    _assert_same_rows(got, orc.hash_join(orc.JoinSpec(orc.JOIN_INNER, [0], [0], [orc.T_INT64]), outer, inner))
    assert "join_fast_table_init" in launches and "join_fast_insert" in launches, launches
    assert not any(k.startswith("join_fast_build_") for k in launches), launches


# ------------------------------------------------------------------------------------------------ crafted keys
@pytest.mark.parametrize("block,share", [(16, 0.5), (2, 0.25)], ids=["block16", "block2"])
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_build_rows_leaving_their_block(gu, radix, jt, block, share):
    """Build keys whose home slot is the last slot of their block: most rows run off the end of their block and are
    inserted afterwards into the finished table (the last block's ones wrap to slot 0).  With 2-slot blocks a split
    CTA's partitions also cover more blocks than it places directly, so rows are deferred by the split as well.
    `share`: the least fraction of the build rows that run off their block's end."""
    radix.setenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", str(block))
    nb = 20_000
    keys, leaving = _crafted_keys(nb, block, 2, 64 << 10, seed=31 + block)
    assert leaving > share * nb
    outer, inner = _crafted_tables(keys, 60_000, seed=50 + jt)
    got, info = _join(gu, jt, outer, inner)
    P, nslots = table_geometry(nb, 2, 64 << 10)
    assert info.fast_path == 1 and info.partitions == P and info.table_slots == nslots
    _assert_same_rows(got, orc.hash_join(orc.JoinSpec(jt, [0], [0], [orc.T_INT64]), outer, inner))


@pytest.mark.parametrize("case", ["duplicate", "key_empty"])
def test_build_crafted_keys_fall_back(gu, radix, case):
    """A duplicated crafted key (both copies leave their block, or one of them does) and KEY_EMPTY as a build key
    make the build hand over to the generic chained path; the result is still the oracle's."""
    radix.setenv("GSQL_JOIN_BUILD_BLOCK_SLOTS", "16")
    keys, _ = _crafted_keys(20_000, 16, 2, 64 << 10, seed=77)
    if case == "duplicate":
        keys = np.concatenate([keys, keys[[5, 1234, 19_999]]])
    else:
        keys = np.concatenate([keys[:10_000], [KEY_EMPTY], keys[10_000:]]).astype(np.int64)
    outer, inner = _crafted_tables(keys, 40_000, seed=88)
    if case == "key_empty":
        outer[0][0][:3] = KEY_EMPTY
    got, info = _join(gu, orc.JOIN_INNER, outer, inner)
    assert info.fast_path == 0
    _assert_same_rows(got, orc.hash_join(orc.JoinSpec(orc.JOIN_INNER, [0], [0], [orc.T_INT64]), outer, inner))


# ------------------------------------------------------------------------------------------------ which kernels run
def test_build_kernel_selection(gu, radix):
    """Radix mode builds with the split, slab and deferred-insert kernels (k_fj_build_split, k_fj_build_slab and
    k_fj_insert, launched as join_fast_build_split / _slab / _deferred) and never EMPTY-fills the table separately."""
    outer, inner = _tables(20_000, 50_000, np.int64, [np.int32, np.int32], [np.int32, np.int32], seed=5)
    launches = {}
    got, info = _join(gu, orc.JOIN_INNER, outer, inner, launches)
    assert info.fast_path == 1 and info.partitions > 1
    _assert_same_rows(got, orc.hash_join(orc.JoinSpec(orc.JOIN_INNER, [0], [0], [orc.T_INT64]), outer, inner))
    expect = {"join_fast_hist_build", "join_fast_scatter_build", "join_fast_build_split", "join_fast_build_slab", "join_fast_build_deferred"}
    assert {k for k in launches if k.startswith("join_fast_") and not k.startswith("join_fast_scan")} == expect, launches
