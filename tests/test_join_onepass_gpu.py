"""The radix join's one-pass probe partitioning: k_fj_scatter_sm writes each probe partition into a fixed region of the
packed buffer, reserving space in blocks of K rows, and the probe skips the KEY_EMPTY gap rows.  Every case is compared
with the CPU oracle as a row multiset, and the kernel profile shows which layout ran: the one-pass layout has no
probe-side histogram; a region that overflows (skewed keys) or a probe key equal to KEY_EMPTY re-runs the batch on the
exact layout.  Run on an H100 with `pytest -m gpu`.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import kat_util as ku
from tests.test_join_scatter_gpu import LAYOUTS, _assert_same_rows, _device_view, _tables

pytestmark = pytest.mark.gpu

ALL_JOINS = [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT, orc.JOIN_SEMI, orc.JOIN_ANTI]
C2_PAY = [np.int32, np.int32]
KEY_EMPTY = np.iinfo(np.int64).min


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


@pytest.fixture
def radix(monkeypatch):
    """Radix mode at test sizes (P = 3..11 for 30 000 build rows of W = 1..4) with 16-row reservation blocks, so that
    a ~1 M-row probe batch fits its regions and every partition run crosses blocks."""
    monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(256 << 10))
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    monkeypatch.setenv("GSQL_JOIN_PART_BLOCK_ROWS", "16")
    monkeypatch.delenv("GSQL_JOIN_SUB_BATCH", raising=False)
    return monkeypatch


def _join(gu, jt, outer, inner, kc):
    """Runs the join with the context's kernel profile on; returns (rows, partitions, profiled kernel names)."""
    from galaxysql_b200 import api
    ctx = gu.ctx()
    kt = orc.T_INT32 if outer[kc][0].dtype == np.int32 else orc.T_INT64
    j = api.HashJoin(ctx, jt, gu._types(outer), gu._types(inner), [kc], [0], [kt])
    try:
        j.build_consume(gu.to_device(inner))
        j.build_finish()
        info = j.info()
        assert info.fast_path == 1 and info.partitions > 1
        ctx.profile(True)
        ctx.profile_reset()
        try:
            got = gu.to_numpy(j.probe(_device_view(outer, 0)))
            names = set(ctx.profile_dump())
        finally:
            ctx.profile(False)
    finally:
        j.close()
    return got, info.partitions, names


def _check(gu, jt, outer, inner, kc, onepass):
    got, P, names = _join(gu, jt, outer, inner, kc)
    ran_onepass = "join_fast_gaps_probe" in names and "join_fast_hist_probe" not in names
    if onepass:
        assert ran_onepass, sorted(names)
    else:  # spilled: the one-pass attempt, then the exact path
        assert "join_fast_gaps_probe" in names and "join_fast_hist_probe" in names, sorted(names)
    spec = orc.JoinSpec(jt, [kc], [0], [orc.T_INT32 if outer[kc][0].dtype == np.int32 else orc.T_INT64])
    _assert_same_rows(got, orc.hash_join(spec, outer, inner))
    return P


def _partition_of(keys, P):
    """part_of(key_hash(k), P) of join_fast.cuh, for BIGINT keys."""
    k = keys.astype(np.int64).view(np.uint64)
    h = (k ^ (k >> np.uint64(32))) * np.uint64(0x9E3779B97F4A7C15)
    return ((h >> np.uint64(32)) * np.uint64(P)) >> np.uint64(32)


# ------------------------------------------------------------------------------------------------ widths, join types
@pytest.mark.parametrize("key_dtype", [np.int64, np.int32], ids=["bigint_key", "int_key"])
@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("jt", ALL_JOINS)
def test_onepass_widths_and_join_types(gu, radix, jt, W, key_dtype):
    """W = 1..4 packed words, INT32 and BIGINT keys, all five join types: gap rows are never emitted, not even as
    unmatched LEFT / RIGHT / ANTI rows.  1 000 003 probe rows: the last tile is ragged."""
    bp, pp = LAYOUTS[W]
    kc = 1 if pp else 0
    outer, inner = _tables(30_000, 1_000_003, key_dtype, bp, pp, seed=500 + 10 * W + (key_dtype == np.int32), probe_key_col=kc)
    _check(gu, jt, outer, inner, kc, onepass=True)


# ------------------------------------------------------------------------------------------------ reservation blocks
@pytest.mark.parametrize("jt", [orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_onepass_runs_within_and_across_blocks(gu, radix, jt):
    """C2 layout, P = 72, 128-row blocks against ~85-row runs per tile and partition: runs that stay in the current
    block, runs that continue in the reserved next block, and the occasional run longer than the room left plus one
    block.  24 M probe rows, so that two blocks per CTA and partition stay within the 1/8 padding limit; ~2700 build
    keys per partition, so that partition sizes stay within the regions' spread allowance."""
    radix.setenv("GSQL_JOIN_PART_BYTES", str(128 << 10))  # 196 608 build rows -> P = 72
    radix.setenv("GSQL_JOIN_PART_BLOCK_ROWS", "128")
    outer, inner = _tables(196_608, 24_000_017, np.int64, C2_PAY, C2_PAY, seed=41)
    assert _check(gu, jt, outer, inner, 0, onepass=True) == 72


def test_onepass_partitions_near_max_p(gu, radix):
    """P = MAX_P (1024) with one-row blocks: every run takes a reservation of its own size.  ~7800 build keys per
    partition keep the partition sizes within the regions' spread allowance."""
    radix.setenv("GSQL_JOIN_PART_BYTES", "370000")  # 8 M build rows -> P = 1024
    radix.setenv("GSQL_JOIN_PART_BLOCK_ROWS", "1")
    outer, inner = _tables(8_000_000, 12_000_001, np.int64, C2_PAY, C2_PAY, seed=42)
    assert _check(gu, orc.JOIN_INNER, outer, inner, 0, onepass=True) == 1024


# ------------------------------------------------------------------------------------------------ exact fallback
@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI])
def test_onepass_single_key_overflows(gu, radix, jt):
    """Every probe row carries the same key: its partition's region overflows and the batch is joined again from the
    exact layout, once."""
    outer, inner = _tables(30_000, 1_000_003, np.int64, C2_PAY, C2_PAY, seed=43)
    outer[0] = (np.full(len(outer[0][0]), inner[0][0][7], dtype=np.int64), None)
    _check(gu, jt, outer, inner, 0, onepass=False)


@pytest.mark.parametrize("jt", [orc.JOIN_INNER, orc.JOIN_RIGHT])
def test_onepass_hot_partition_overflows(gu, radix, jt):
    """Half of the probe rows fall into partition 0 (distinct keys, found by restating the hash): its region
    overflows and the exact path runs."""
    outer, inner = _tables(30_000, 1_000_003, np.int64, C2_PAY, C2_PAY, seed=44)
    keys = inner[0][0]
    hot = keys[_partition_of(keys, 6) == 0]  # 90 000 slots of 16 B in 256 KB partitions: P = 6
    assert len(hot) > 100
    pk = outer[0][0].copy()
    half = np.arange(len(pk)) % 2 == 0
    pk[half] = hot[(ku.rand_u64(int(half.sum()), 45) % np.uint64(len(hot))).astype(np.int64)]
    outer[0] = (pk, None)
    assert _check(gu, jt, outer, inner, 0, onepass=False) == 6


@pytest.mark.parametrize("jt", [orc.JOIN_LEFT, orc.JOIN_ANTI, orc.JOIN_INNER])
def test_onepass_sentinel_probe_key(gu, radix, jt):
    """Probe keys equal to KEY_EMPTY (the BIGINT minimum) would read as gap rows: the batch takes the exact layout and
    those rows come out unmatched, as before."""
    outer, inner = _tables(30_000, 1_000_003, np.int64, C2_PAY, C2_PAY, seed=46)
    pk = outer[0][0].copy()
    pk[::1001] = KEY_EMPTY
    outer[0] = (pk, None)
    _check(gu, jt, outer, inner, 0, onepass=False)
