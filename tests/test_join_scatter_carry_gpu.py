"""The radix scatter's sector carry (k_fj_scatter_sm, W = 2): a partition run that would end inside a 32-byte sector holds
its last row back and writes it at the front of the partition's run in the CTA's next tile, so that no flushed run ends
mid-sector.  Each case gives every CTA several tiles, so that rows are held back many times, and is compared with the CPU
oracle as a row multiset under INNER, LEFT and ANTI, on both probe layouts and through a region overflow that leaves the
kernel with rows still held.  Run on an H100 with `pytest -m gpu`.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import kat_util as ku
from tests.test_join_onepass_gpu import _check, _join, _partition_of
from tests.test_join_scatter_gpu import _assert_same_rows, _tables

pytestmark = pytest.mark.gpu

JOIN_TYPES = [orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_ANTI]
C2_PAY = [np.int32, np.int32]  # BIGINT key + 2 INT: W = 2 on both sides
ROWS = 132 * 6144 * 3 + 4321  # three and a bit 6144-row tiles per CTA on a 132-SM H100


@pytest.fixture(scope="module")
def gu():
    from tests import gpu_util
    gpu_util.ctx()  # raises loudly if the extension or the device is missing — no CPU fallback
    return gpu_util


@pytest.fixture
def radix(monkeypatch):
    """Radix mode at test sizes (P = 6 for 30 000 C2 build rows) with 16-row reservation blocks."""
    monkeypatch.setenv("GSQL_JOIN_PART_BYTES", str(256 << 10))
    monkeypatch.setenv("GSQL_JOIN_PART_MIN_ROWS", "0")
    monkeypatch.setenv("GSQL_JOIN_PART_BLOCK_ROWS", "16")
    monkeypatch.delenv("GSQL_JOIN_SUB_BATCH", raising=False)
    return monkeypatch


@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_carry_exact_layout_many_tiles(gu, radix, jt):
    """2^20-row blocks push the probe side onto the exact layout, whose per-CTA offsets start at odd rows as often as
    at even ones; P = 72 gives ~85-row runs per tile, half of them odd."""
    radix.setenv("GSQL_JOIN_PART_BLOCK_ROWS", str(1 << 20))
    radix.setenv("GSQL_JOIN_PART_BYTES", str(128 << 10))  # 196 608 build rows -> P = 72
    outer, inner = _tables(196_608, ROWS, np.int64, C2_PAY, C2_PAY, seed=1500 + jt)
    got, P, names = _join(gu, jt, outer, inner, 0)
    assert "join_fast_hist_probe" in names and "join_fast_gaps_probe" not in names, sorted(names)
    assert P == 72
    _assert_same_rows(got, orc.hash_join(orc.JoinSpec(jt, [0], [0], [orc.T_INT64]), outer, inner))


@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_carry_regions_many_tiles(gu, radix, jt):
    """One-pass regions, 16-row blocks: runs continue in the next block or in a fresh reservation, and a held row
    always lies just before the partition's next row."""
    outer, inner = _tables(30_000, ROWS, np.int64, C2_PAY, C2_PAY, seed=1600 + jt)
    _check(gu, jt, outer, inner, 0, onepass=True)


@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_carry_region_overflow(gu, radix, jt):
    """Half of the probe rows fall into partition 0: its region overflows after CTAs have held rows back, the batch
    runs again on the exact layout, and no held row is lost or written twice."""
    outer, inner = _tables(30_000, ROWS, np.int64, C2_PAY, C2_PAY, seed=1700 + jt)
    keys = inner[0][0]
    hot = keys[_partition_of(keys, 6) == 0]  # 90 000 slots of 16 B in 256 KB partitions: P = 6
    pk = outer[0][0].copy()
    half = np.arange(len(pk)) % 2 == 0
    pk[half] = hot[(ku.rand_u64(int(half.sum()), 1701 + jt) % np.uint64(len(hot))).astype(np.int64)]
    outer[0] = (pk, None)
    assert _check(gu, jt, outer, inner, 0, onepass=False) == 6
