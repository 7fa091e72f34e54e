"""tests/exchange_ref.py (the exchange's routing by definition) against hand-worked values of the Java functions it
restates and against the CPU oracle (oracle.c) on every seeded case; the wire format's page rules against
oracle/serde.py.  No GPU."""
import struct

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import serde as oserde
from tests import exchange_cases as xc
from tests import exchange_ref as xr
from tests import wire_cases as wc
from tests.hash_join_ref import rows_bits

INT_MIN = -2**31


def _f64(bits):
    return np.array([bits], dtype=np.uint64).view(np.float64)


# ------------------------------------------------------------------------------------------------ Java KATs
def test_long_hash_code():
    # Long.hashCode(v) = (int)(v ^ (v >>> 32))
    # -1L:      0xFFFFFFFF_FFFFFFFF ^ 0x00000000_FFFFFFFF = 0xFFFFFFFF_00000000 -> (int) 0
    # 1L << 32: 0x00000001_00000000 ^ 0x00000000_00000001 = 0x00000001_00000001 -> (int) 1
    # MIN:      0x80000000_00000000 ^ 0x00000000_80000000 -> (int) 0x80000000
    assert xr.long_hash([-1, 1 << 32, -2**63, 5]).tolist() == [0, 1, INT_MIN, 5]


def test_double_hash_code():
    # Double.hashCode(d) = Long.hashCode(doubleToLongBits(d))
    # -0.0: bits 0x80000000_00000000 -> 0x80000000 = Integer.MIN_VALUE; +0.0 -> 0
    # NaN (any bits) -> 0x7FF80000_00000000 -> low word 0 ^ high word 0x7FF80000 = 2146959360
    # 1.0: 0x3FF00000_00000000 -> 0x3FF00000 = 1072693248
    neg0, pos0 = _f64(0x8000000000000000), _f64(0)
    assert xr.block_hash((neg0, None), xc.F64).tolist() == [INT_MIN]
    assert xr.block_hash((pos0, None), xc.F64).tolist() == [0]
    nans = xc.f64_array(xc.NANS)
    assert xr.block_hash((nans, None), xc.F64).tolist() == [2146959360] * len(xc.NANS)
    assert xr.block_hash((np.array([1.0]), None), xc.F64).tolist() == [1072693248]


def test_widening_and_null_hash():
    # INT -> BIGINT sign-extends: -1 -> -1L -> Long.hashCode 0; INT -> DOUBLE: 1 -> 1.0 -> 1072693248
    neg = np.array([-1, 7], dtype=np.int32)
    assert xr.block_hash((neg, None), xc.I32).tolist() == [-1, 7]
    assert xr.block_hash((neg, None), xc.I64).tolist() == [0, 7]
    assert xr.block_hash((np.array([1], np.int32), None), xc.F64).tolist() == [1072693248]
    # BIGINT -> DOUBLE rounds to nearest even: 2^53 + 1 -> 2^53 (bits 0x43400000_00000000 -> 0x43400000)
    assert xr.block_hash((np.array([2**53 + 1, 2**53], np.int64), None), xc.F64).tolist() == [0x43400000] * 2
    # a NULL hashes to 0 whatever its value bits
    assert xr.block_hash((np.array([5, 6], np.int64), np.array([True, False])), xc.I64).tolist() == [0, 6]
    with pytest.raises(xr.Unsupported):
        xr.block_hash((np.array([1], np.int64), None), xc.I32)


def test_chunk_hash_code():
    # Chunk.hashCode: h = 31 * h + block hash, from 0.  (INT 3, BIGINT 1L << 32) -> 31 * 3 + 1 = 94; zero channels -> 0
    cols = [(np.array([3], np.int32), None), (np.array([1 << 32], np.int64), None)]
    assert xr.row_hash(cols, [0, 1]).tolist() == [94]
    assert xr.row_hash(cols, []).tolist() == [0]
    # wraparound: 31 * 0x7FFFFFFF + 0 = 0xF_7FFFFFE1 -> (int) 0x7FFFFFE1 = 2147483617;
    #             31 * 0x7FFFFFFF + 0x10000000 = 0xF_8FFFFFE1 -> (int) 0x8FFFFFE1 = -1879048223
    big = (np.array([2**31 - 1] * 2, np.int32), None)
    assert xr.row_hash([big, (np.array([0, 1 << 28], np.int32), None)], [0, 1]).tolist() == [2147483617, -1879048223]


def test_murmur_hash3_and_partition():
    # fastutil murmurHash3(x): x ^= x >>> 16; x *= 0x85ebca6b; x ^= x >>> 13; x *= 0xc2b2ae35; x ^= x >>> 16
    # 0 -> 0, as every step keeps 0; the other pins follow the Java source line by line in 32-bit ints (mm below)
    def mm(x):
        x &= 0xFFFFFFFF
        x ^= x >> 16
        x = (x * 0x85EBCA6B) & 0xFFFFFFFF
        x ^= x >> 13
        x = (x * 0xC2B2AE35) & 0xFFFFFFFF
        x ^= x >> 16
        return x - (1 << 32) if x >= 1 << 31 else x
    pins = {0: 0, 1: 1364076727, -1: -2114883783, 42: 142593372, INT_MIN: 1832674720, 2146959360: 104869765}
    for x, m in pins.items():
        assert mm(x) == m
        assert int(xr.murmur_hash3([x])[0]) == m
    # ExecUtils.partition: n a power of two -> m & (n - 1); else (m & Integer.MAX_VALUE) % n
    #   h = 1,  n = 8:    1364076727 & 7 = 7
    #   h = 1,  n = 3:    1364076727 % 3 = 1
    #   h = -1, n = 10:   (-2114883783 & 0x7FFFFFFF) = 32599865 -> % 10 = 5
    #   h = 42, n = 1000: 142593372 % 1000 = 372
    #   h = NaN's hash, n = 1024: 104869765 & 1023 = 901
    for (h, n), p in {(1, 8): 7, (1, 3): 1, (-1, 10): 5, (42, 1000): 372, (2146959360, 1024): 901, (INT_MIN, 6): 4}.items():
        assert int(xr.partition([h], n)[0]) == p
        assert orc.partition(h, n) == p


def test_round_robin_rule():
    cols = [(np.zeros(10, np.int64), None)]
    assert xr.destinations(cols, [0], 4, mode=xr.RANDOM).tolist() == [0, 1, 2, 3, 0, 1, 2, 3, 0, 1]
    assert xr.destinations(cols, [0], 3, mode=xr.RANDOM, row_base=5).tolist() == [2, 0, 1, 2, 0, 1, 2, 0, 1, 2]


# ------------------------------------------------------------------------------------------------ reference vs oracle
CASES = xc.all_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_reference_matches_oracle(case):
    cols, ch, kt, n = case["cols"], case["channels"], case["key_types"], case["nparts"]
    h = xr.row_hash(cols, ch, kt)
    if ch:
        assert np.array_equal(h, orc.hash_rows([cols[c] for c in ch], kt))
    else:
        assert not h.any()
    dest = xr.partition(h, n)
    assert np.array_equal(dest, orc.partition_ids(h, n))
    if not ch or not len(cols[0][0]):
        return  # the oracle's exchange needs a key and a row
    ocols, ocounts = orc.partition_exchange(cols, ch, n, kt)
    assert ocounts.tolist() == xr.counts(dest, n).tolist()
    assert xr.grouped_rows(ocols, ocounts) == xr.routed_rows(cols, dest)


def test_cases_reach_every_shape():
    ids = [c["id"] for c in CASES]
    assert {c["nparts"] for c in CASES} == set(xc.NPARTS)
    assert {len(c["channels"]) for c in CASES} == {0, 1, 2, 3, 8}
    assert {len(c["cols"][0][0]) for c in CASES} >= set(xc.ROWS) | {xc.BIG_ROWS}
    assert len(ids) == len(set(ids))


# ------------------------------------------------------------------------------------------------ wire format rules
def test_zero_row_page_bytes():
    # a 0-row page of two columns: frame (0, UNCOMPRESSED, 12, 12), blockCount 2, two blocks of positionCount 0, no bits
    b = oserde.serialize_pages([(np.zeros(0, np.int64), None), (np.zeros(0, np.int32), None)], [1, 0], [0])
    assert b == struct.pack("<ibii", 0, 0, 12, 12) + struct.pack("<iii", 2, 0, 0)
    back = oserde.deserialize(b, [1, 0])
    assert [len(v) for v, _ in back] == [0, 0]


def test_java_shaped_pages_round_trip():
    n = sum(wc.JAVA_PAGE_SIZES)
    cols = [xc.table(n, 5, 0.3)[k] for k in (0, 2, 6)]
    types = [xc.I32, xc.F64, xc.I64]
    b = oserde.serialize_pages(cols, types, wc.JAVA_PAGE_SIZES)
    assert [m for _, m, _ in wc.pages(b, types)] == wc.JAVA_PAGE_SIZES
    assert rows_bits(oserde.deserialize(b, types)) == rows_bits(cols)
    # equal page sizes give the bytes of serialize()
    assert oserde.serialize_pages(cols, types, [1000] * (n // 1000) + [n % 1000]) == oserde.serialize(cols, types, 1000)


def test_trailing_bytes_inside_a_page_are_ignored():
    good, types, cols = wc.two_page_stream(xc.I64)
    for page in (0, 1):
        b = wc.with_trailing_bytes(good, types, page, b"\xff" * 11)
        dec = oserde.deserialize(b, types)
        assert rows_bits(dec) == rows_bits(cols)


@pytest.mark.parametrize("last_type", [xc.I32, xc.I64])
def test_corrupt_streams_are_refused(last_type):
    for name, b, types, _ in wc.corrupt_streams(last_type):
        with pytest.raises(oserde.WireFormatError):
            oserde.deserialize(b, types)
