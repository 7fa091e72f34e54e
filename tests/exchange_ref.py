"""The exchange's routing by definition: which consumer a row goes to, restated in numpy with int32 wraparound.

This is the yardstick the exchange tests hold the GPU (gsql_hash_rows, gsql_xchg_partition, gsql_xchg_push,
gsql_xchg_all_to_all) and the CPU oracle (oracle.c) against.  It shares no code with either.  The rules, from the
reference (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):

* A key column is first converted to its unified type (EX/chunk/Converters.java): INT stays INT, INT -> BIGINT
  sign-extends, INT or BIGINT -> DOUBLE is Java's ``(double)`` cast (round to nearest, ties to even).  Narrowing targets
  (BIGINT -> INT, DOUBLE -> an integer) go through DataTypeUtils.convert, which is not restated here: they raise
  Unsupported.
* Block.hashCode(position): a NULL hashes to 0; INT is the value; BIGINT is Long.hashCode = (int)(v ^ (v >>> 32));
  DOUBLE is Long.hashCode(Double.doubleToLongBits(d)): every NaN becomes 0x7ff8000000000000, -0.0 keeps its sign bit.
* Chunk.hashCode(position): h = 31 * h + block hash over the channels, from h = 0 (so zero channels give 0).
* ExecUtils.partition(h, n): m = fastutil HashCommon.murmurHash3(h); m & (n - 1) for a power-of-two n, else
  (m & Integer.MAX_VALUE) % n.
* GSQL_XCHG_RANDOM (round-robin): destination = row index mod n, the row index counted over the caller's whole batch.
"""
from __future__ import annotations

from collections import Counter
from typing import List, Optional, Sequence, Tuple

import numpy as np

from tests.hash_join_ref import rows_bits

Col = Tuple[np.ndarray, Optional[np.ndarray]]

T_INT32, T_INT64, T_FP64 = 0, 1, 2
HASH, BROADCAST, RANDOM = 0, 1, 2
CANONICAL_NAN = 0x7FF8000000000000
_T_OF = {np.dtype(np.int32): T_INT32, np.dtype(np.int64): T_INT64, np.dtype(np.float64): T_FP64}


class Unsupported(ValueError):
    """A key conversion this restatement does not cover (a narrowing one)."""


def long_hash(v) -> np.ndarray:
    """Long.hashCode: (int)(v ^ (v >>> 32)), as int32."""
    u = np.asarray(v, dtype=np.int64).view(np.uint64)
    return (u ^ (u >> np.uint64(32))).astype(np.uint32).view(np.int32)


def double_bits(d) -> np.ndarray:
    """Double.doubleToLongBits: the IEEE bits, every NaN canonicalised."""
    d = np.asarray(d, dtype=np.float64)
    return np.where(np.isnan(d), np.int64(CANONICAL_NAN), d.view(np.int64))


def block_hash(col: Col, unified_type: int) -> np.ndarray:
    """Block.hashCode of every row of `col` after its conversion to `unified_type`."""
    data, nulls = col
    data = np.asarray(data)
    src = _T_OF[data.dtype]
    if unified_type == T_INT32:
        if src != T_INT32:
            raise Unsupported("narrowing key conversion to INT")
        h = data.astype(np.int32)
    elif unified_type == T_INT64:
        if src == T_FP64:
            raise Unsupported("narrowing key conversion DOUBLE -> BIGINT")
        h = long_hash(data.astype(np.int64))
    else:
        h = long_hash(double_bits(data.astype(np.float64)))  # (double) cast: round to nearest
    if nulls is not None:
        h = np.where(np.asarray(nulls).astype(bool), np.int32(0), h)
    return np.asarray(h, dtype=np.int32)


def row_hash(cols: Sequence[Col], channels: Sequence[int], key_types: Optional[Sequence[int]] = None) -> np.ndarray:
    """Chunk.hashCode of every row over `channels` (h = 31 * h + block hash, int32 wraparound)."""
    n = len(cols[0][0]) if cols else 0
    kt = list(key_types) if key_types is not None else [_T_OF[np.asarray(cols[c][0]).dtype] for c in channels]
    h = np.zeros(n, dtype=np.uint32)
    for c, t in zip(channels, kt):
        h = h * np.uint32(31) + block_hash(cols[c], t).view(np.uint32)
    return h.view(np.int32)


def murmur_hash3(x) -> np.ndarray:
    """fastutil HashCommon.murmurHash3(int)."""
    h = np.asarray(x, dtype=np.int32).view(np.uint32).copy()
    h ^= h >> np.uint32(16)
    h *= np.uint32(0x85EBCA6B)
    h ^= h >> np.uint32(13)
    h *= np.uint32(0xC2B2AE35)
    h ^= h >> np.uint32(16)
    return h.view(np.int32)


def partition(h, nparts: int) -> np.ndarray:
    """ExecUtils.partition(hash, n)."""
    m = murmur_hash3(h).view(np.uint32)
    if nparts & (nparts - 1) == 0:
        return (m & np.uint32(nparts - 1)).astype(np.int32)
    return ((m & np.uint32(0x7FFFFFFF)) % np.uint32(nparts)).astype(np.int32)


def destinations(cols: Sequence[Col], channels: Sequence[int], nparts: int, key_types: Optional[Sequence[int]] = None,
                 mode: int = HASH, row_base: int = 0) -> np.ndarray:
    """Destination of every row: ExecUtils.partition(Chunk.hashCode) for HASH, row index mod nparts for RANDOM."""
    n = len(cols[0][0]) if cols else 0
    if mode == RANDOM:
        return ((np.arange(n, dtype=np.int64) + row_base) % nparts).astype(np.int32)
    if mode != HASH:
        raise Unsupported("broadcast has no per-row destination")
    return partition(row_hash(cols, channels, key_types), nparts)


def take(cols: Sequence[Col], mask: np.ndarray) -> List[Col]:
    return [(np.asarray(d)[mask], None if nl is None else np.asarray(nl).astype(bool)[mask]) for d, nl in cols]


def counts(dest: np.ndarray, nparts: int) -> np.ndarray:
    """Rows per destination."""
    return np.bincount(np.asarray(dest, dtype=np.int64), minlength=nparts).astype(np.int64)


def routed_rows(cols: Sequence[Col], dest: np.ndarray) -> Counter:
    """Multiset of (destination, row...) with rows compared bit for bit (hash_join_ref.rows_bits: a DOUBLE by its 64-bit
    pattern, a NULL's value ignored)."""
    return rows_bits([(np.asarray(dest, dtype=np.int64), None)] + list(cols))


def grouped_rows(cols: Sequence[Col], part_counts: Sequence[int]) -> Counter:
    """routed_rows of an exchange's output, whose destination p holds rows [sum(counts[:p]), +counts[p])."""
    dest = np.repeat(np.arange(len(part_counts), dtype=np.int64), np.asarray(part_counts, dtype=np.int64))
    assert len(dest) == (len(cols[0][0]) if cols else 0), "part counts do not add up to the output's rows"
    return routed_rows(cols, dest)
