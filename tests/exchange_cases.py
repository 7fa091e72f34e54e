"""Seeded exchange cases shared by test_exchange_ref_cpu.py (reference vs oracle) and test_exchange_gpu.py (GPU vs
reference): every key shape, key widening, NULL density and special value the routing has to hash exactly, at the
part counts and row counts where a partition kernel goes wrong.

A case is a dict: ``id``, ``cols`` (the batch; every column travels), ``channels`` / ``key_types`` (the partition
key and its unified types) and ``nparts``.
"""
from __future__ import annotations

from typing import List

import numpy as np

from tests import kat_util as ku
from tests.join_cases import FINITE_SPECIALS, NANS, NEG_ZERO, POS_ZERO, f64_array, pick

I32, I64, F64 = 0, 1, 2
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
MAX_PARTS = 1024

NPARTS = [1, 2, 3, 6, 8, 10, 64, 1000, MAX_PARTS]
ROWS = [0, 1, 255, 256, 257, 4097]
BIG_ROWS = 300_007          # several 256-row chunks per partition block, and several blocks
NULL_FRACS = [0.0, 0.03, 1.0]

SPECIAL_F64 = f64_array(NANS + FINITE_SPECIALS + [NEG_ZERO, POS_ZERO] + [0x4340000000000001, 0xC3E0000000000000])
INT32_EDGES = np.array([INT32_MIN, INT32_MIN + 1, -1, 0, 1, INT32_MAX], dtype=np.int32)
INT64_EDGES = np.array([INT64_MIN, INT64_MIN + 1, -1, 0, 1, INT64_MAX, 1 << 32, -(1 << 32), (1 << 53) + 1, (1 << 62) + 3,
                        -(1 << 53) - 1, 0xFFFFFFFF], dtype=np.int64)


def _mix(values: np.ndarray, random: np.ndarray, seed: int) -> np.ndarray:
    """About a quarter of the rows drawn from `values` (edge values), the rest from `random`."""
    n = len(random)
    if n == 0:
        return random
    edge, _ = pick(values, n, seed)
    use = (ku.rand_u64(n, seed, stream=3) % np.uint64(4)) == 0
    return np.where(use, edge, random).astype(random.dtype)


def table(n: int, seed: int, null_frac: float) -> List["ku.Col"]:
    """The batch every case routes (key columns are among its columns):

    0 INT32   edge values and small integers (repeats)       NULLs at null_frac
    1 BIGINT  edge values and 40-bit integers                NULLs at null_frac
    2 DOUBLE  NaNs with payloads, +-0.0, +-Inf, subnormals   NULLs at null_frac
    3 INT32   negative values (sign extension under BIGINT)  NULLs at null_frac
    4 BIGINT  above 2^53 (rounded by the (double) cast)      NULLs at null_frac
    5 DOUBLE  special values, no NULL mask (payload)
    6 BIGINT  random bits, NULLs at 30 % (payload)
    7 INT32   row index (payload: makes rows distinct)
    """
    r = lambda s: ku.rand_u64(n, seed + s)  # noqa: E731
    c0 = _mix(INT32_EDGES, ((r(0) % np.uint64(1000)).astype(np.int64) - 500).astype(np.int32), seed + 100)
    c1 = _mix(INT64_EDGES, (r(1) % np.uint64(1 << 40)).astype(np.int64) - (1 << 39), seed + 101)
    c2 = _mix(SPECIAL_F64, (r(2) % np.uint64(1000)).astype(np.float64) / 8.0 - 60.0, seed + 102)
    c3 = _mix(INT32_EDGES[:3], -(r(3) % np.uint64(1 << 31)).astype(np.int64).astype(np.int32) - 1, seed + 103)
    c4 = _mix(INT64_EDGES, ((r(4) >> np.uint64(2)) | np.uint64(1 << 53)).astype(np.int64), seed + 104)
    c5 = pick(SPECIAL_F64, n, seed + 105)[0]
    c6 = r(6).view(np.int64)
    c7 = np.arange(n, dtype=np.int32)
    nf = lambda d, s: ku.with_nulls(d, null_frac, seed + 200 + s)  # noqa: E731
    return [nf(c0, 0), nf(c1, 1), nf(c2, 2), nf(c3, 3), nf(c4, 4), (c5, None), ku.with_nulls(c6, 0.3, seed + 206), (c7, None)]


# (name, channels, unified key types): 0, 1, 2, 3 and 8 channels; every widening
KEYS = [
    ("none", [], []),
    ("i32", [0], [I32]),
    ("i64", [1], [I64]),
    ("f64", [2], [F64]),
    ("i32_as_i64", [3], [I64]),
    ("i32_as_f64", [0], [F64]),
    ("i64_as_f64", [4], [F64]),
    ("i32_f64", [0, 2], [I32, F64]),
    ("i64_i32w_f64", [1, 3, 2], [I64, I64, F64]),
    ("eight", [0, 1, 2, 3, 4, 5, 6, 0], [I32, I64, F64, I64, F64, F64, I64, F64]),
]
KEY_OF = {k[0]: k for k in KEYS}


def case(id_, cols, key, nparts) -> dict:
    name, channels, key_types = KEY_OF[key]
    return dict(id=id_, cols=cols, channels=list(channels), key_types=list(key_types), nparts=nparts)


def key_cases() -> List[dict]:
    """Every key shape at every NULL density, 4097 rows, the part counts taken in turn."""
    out = []
    i = 0
    for k, (name, _, _) in enumerate(KEYS):
        for f in NULL_FRACS:
            nparts = NPARTS[i % len(NPARTS)]
            i += 1
            out.append(case(f"key-{name}-null{int(f * 100)}-p{nparts}", table(4097, 1000 + 10 * k, f), name, nparts))
    return out


def shape_cases() -> List[dict]:
    """Every part count at every small row count (tile edges: 255 / 256 / 257, 4097), three-channel mixed key."""
    return [case(f"shape-p{p}-n{n}", table(n, 7 + n, 0.03), "i64_i32w_f64", p) for p in NPARTS for n in ROWS]


def big_cases() -> List[dict]:
    """About 300 k rows: many chunks per partition block, and the largest part counts."""
    return [case(f"big-{key}-p{p}", table(BIG_ROWS, 77 + p, 0.03), key, p)
            for key, p in [("eight", 3), ("i64", 8), ("f64", 1000), ("i32_as_i64", MAX_PARTS), ("none", 10)]]


def all_cases() -> List[dict]:
    return key_cases() + shape_cases() + big_cases()
