"""Reference restatement of the runtime bloom filter (test infrastructure, numpy only), independent of the CUDA code:

* XXH64 (seed 0) of one long's 8 little-endian bytes — what the reference's streaming XxHash_64Hasher produces for
  Chunk.ChunkRow.hashCode over one key column (IStreamingHasher.putInt -> putLong; DoubleBlock puts doubleToRawLongBits;
  a NULL puts NULL_VALUE 0);
* BloomFilter.put64 / mightContain64 (polardbx-common .../utils/bloomfilter/BloomFilter.java:65-76, :114-129) over a
  long[numBits/64] bitmap (BitSet.java:53-82);
* the sizing of RuntimeFilterBuilderExecFactory.java:75-98 + RuntimeFilterUtil.findMinFpp + BloomFilter.createEmpty
  (BloomFilterUtil.java:46-67).

tests/golden/xxh64_long.json pins the hash to published and libxxhash vectors."""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import numpy as np

P1, P2, P3 = np.uint64(0x9E3779B185EBCA87), np.uint64(0xC2B2AE3D27D4EB4F), np.uint64(0x165667B19E3779F9)
P4, P5 = np.uint64(0x85EBCA77C2B2AE63), np.uint64(0x27D4EB2F165667C5)
DEFAULT_FPP = float(np.float32(0.03))      # BloomFilter.DEFAULT_FPP = 0.03f, widened to double
MIN_SIZE, MAX_SIZE = 1000, 2 * 1024 * 1024  # ConnectionParams.BLOOM_FILTER_MIN_SIZE / BLOOM_FILTER_MAX_SIZE defaults
MAX_BITS = (1 << 31) - 64                   # BloomFilter.java:45 Math.multiplyExact(length, Long.SIZE) must fit an int


def _rotl(x: np.ndarray, r: int) -> np.ndarray:
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def xxh64_long(v) -> np.ndarray:
    """XXH64(seed 0) of the 8 little-endian bytes of each value (int64/uint64 array-like) -> uint64 array."""
    x = np.asarray(v).astype(np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        h = np.full(x.shape, P5 + np.uint64(8), dtype=np.uint64)
        h ^= _rotl(x * P2, 31) * P1
        h = _rotl(h, 27) * P1 + P4
        h ^= h >> np.uint64(33)
        h *= P2
        h ^= h >> np.uint64(29)
        h *= P3
        h ^= h >> np.uint64(32)
    return h


_M64 = (1 << 64) - 1


def xxh64_short(data: bytes, seed: int = 0) -> int:
    """Scalar XXH64 of an input shorter than 32 bytes (the specification's tail path), for the published vectors."""
    assert len(data) < 32
    p1, p2, p3, p4, p5 = (int(p) for p in (P1, P2, P3, P4, P5))
    rotl = lambda x, r: ((x << r) | (x >> (64 - r))) & _M64
    h = (seed + p5 + len(data)) & _M64
    i = 0
    while i + 8 <= len(data):
        k1 = rotl(int.from_bytes(data[i:i + 8], "little") * p2 & _M64, 31) * p1 & _M64
        h = (rotl(h ^ k1, 27) * p1 + p4) & _M64
        i += 8
    if i + 4 <= len(data):
        h = (rotl(h ^ (int.from_bytes(data[i:i + 4], "little") * p1 & _M64), 23) * p2 + p3) & _M64
        i += 4
    while i < len(data):
        h = rotl(h ^ (data[i] * p5 & _M64), 11) * p1 & _M64
        i += 1
    h ^= h >> 33
    h = h * p2 & _M64
    h ^= h >> 29
    h = h * p3 & _M64
    return h ^ (h >> 32)


def xxh64_long_inverse(h: int) -> int:
    """The signed long whose xxh64_long is h: every step of XXH64 over one 8-byte lane is a bijection of 64-bit words
    (odd multiplies, rotations, xor-shifts), so tests can pick keys that reach chosen hash values."""
    p1, p2, p3, p4, p5 = (int(p) for p in (P1, P2, P3, P4, P5))
    inv = lambda p: pow(p, -1, 1 << 64)
    rotr = lambda x, r: ((x >> r) | (x << (64 - r))) & _M64

    def unxorshift(x, s):
        y = x
        for _ in range(64 // s + 1):
            y = x ^ (y >> s)
        return y

    x = unxorshift(h, 32)
    x = x * inv(p3) & _M64
    x = unxorshift(x, 29)
    x = x * inv(p2) & _M64
    x = unxorshift(x, 33)
    x = rotr((x - p4) * inv(p1) & _M64, 27) ^ ((p5 + 8) & _M64)
    v = rotr(x * inv(p1) & _M64, 31) * inv(p2) & _M64
    return v - (1 << 64) if v >> 63 else v


def fastmod_u32(a: int, d: int) -> int:
    """Lemire's exact remainder a % d for 32-bit a and d (M = 2^64 // d + 1 kept mod 2^64), as the kernels compute it."""
    m = (_M64 // d + 1) & _M64
    return (((m * a) & _M64) * d) >> 64


def key_longs(values: np.ndarray, nulls: Optional[np.ndarray] = None) -> np.ndarray:
    """The long the reference's hasher sees per row of a key column: INT sign-extended, BIGINT as is, DOUBLE raw bits,
    NULL -> 0."""
    values = np.asarray(values)
    if values.dtype == np.float64:
        out = values.view(np.int64).copy()
    else:
        out = values.astype(np.int64)
    if nulls is not None:
        out[np.asarray(nulls, bool)] = 0
    return out


def positions(h: np.ndarray, num_bits: int, k: int) -> np.ndarray:
    """(rows, k) bit positions of put64 for hashes h (uint64): combined = (int) h + (int) (h >>> 32), sign bit cleared
    when negative, bit combined % numBits, combined += hash2 — Java int arithmetic as uint32."""
    h = np.asarray(h, dtype=np.uint64)
    h1 = (h & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    h2 = (h >> np.uint64(32)).astype(np.uint32)
    out = np.empty(h.shape + (k,), dtype=np.int64)
    with np.errstate(over="ignore"):
        c = h1 + h2
        for i in range(k):
            c = c & np.uint32(0x7FFFFFFF)
            out[..., i] = c.astype(np.int64) % num_bits
            c = c + h2
    return out


def build(cols: Sequence[Tuple[np.ndarray, Optional[np.ndarray]]], key_col: int, num_bits: int, k: int,
          words: Optional[np.ndarray] = None) -> np.ndarray:
    """BloomFilter.put64 over every row of one key column -> the uint64[num_bits // 64] bitmap (ORed into `words`)."""
    assert num_bits % 64 == 0 and 64 <= num_bits <= MAX_BITS and k >= 1
    words = np.zeros(num_bits // 64, dtype=np.uint64) if words is None else words
    v, nl = cols[key_col]
    pos = np.unique(positions(xxh64_long(key_longs(v, nl)), num_bits, k).ravel())
    np.bitwise_or.at(words, pos >> 6, np.uint64(1) << (pos & 63).astype(np.uint64))
    return words


def might_contain(words: np.ndarray, values: np.ndarray, nulls: Optional[np.ndarray], k: int) -> np.ndarray:
    """mightContain64 per row -> bool array."""
    num_bits = len(words) * 64
    pos = positions(xxh64_long(key_longs(values, nulls)), num_bits, k)
    w = np.asarray(words, dtype=np.uint64)[pos >> 6]
    return (((w >> (pos & 63).astype(np.uint64)) & np.uint64(1)) != 0).all(axis=-1)


def filter_rows(words: np.ndarray, cols, key_col: int, k: int):
    keep = might_contain(words, cols[key_col][0], cols[key_col][1], k)
    return [(d[keep], None if nl is None else np.asarray(nl)[keep]) for d, nl in cols], keep


def _java_int(x: float) -> int:
    """Java's (int) of a double: truncation toward zero, saturating, NaN -> 0."""
    if x != x:
        return 0
    return int(max(min(x, 2147483647.0), -2147483648.0))


def create_empty_sizing(n: int, fpp: float) -> Tuple[int, int]:
    """BloomFilter.createEmpty(method, expectedInsertions, fpp) -> (numBits, numHashFunctions)."""
    p = fpp if fpp != 0 else 5e-324
    nb = _java_int(-n * math.log(p) / (math.log(2) * math.log(2)))
    num_bits = nb + (64 - nb % 64)                                       # nb >= 0 for 0 < p < 1: always adds 1..64 bits
    k = max(1, _java_int(math.floor(num_bits / n * math.log(2) + 0.5)))  # Math.round
    return int(num_bits), k


def sizing(ndv: int, min_size: int = MIN_SIZE, max_size: int = MAX_SIZE) -> Tuple[int, int]:
    """The factory's arithmetic: size = clamp(ndv, min, max), fpp = max(exp(-3.843 size / ndv), DEFAULT_FPP)."""
    size = min(max_size, max(min_size, ndv))
    fpp = DEFAULT_FPP if ndv <= 0 else max(math.exp(-3.843 * size / ndv), DEFAULT_FPP)
    return create_empty_sizing(size, fpp)
