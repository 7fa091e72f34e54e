"""Two restatements of the executor's ORDER BY comparator (EX/utils/ExecUtils.getComparator:451-490), for checking
gsql_sort: a literal one over Python rows with functools.cmp_to_key, and a numpy lexsort form for large inputs.

  * keys compare in order; two NULLs are equal; NULL is the smallest value (OPT/core/datatype/NumberType.compare:110-127);
  * DESC negates the key's result (so NULLs lead under ASC and trail under DESC; OrderByOption.nullLast is never read);
  * INT / BIGINT: natural order; DOUBLE: Double.compareTo (-0.0 < +0.0, every NaN equal and above +Inf).

They sit with the tests so that the C oracle stays unchanged.  Columns are ``(values, nulls)`` numpy pairs, as in api.
"""
from __future__ import annotations

import functools
import math
import struct
from collections import Counter
from typing import List, Optional, Sequence

import numpy as np

T_INT32, T_INT64, T_FP64 = 0, 1, 2


# ------------------------------------------------------------------------------------------------ literal form
def _double_to_long_bits(d: float) -> int:
    """Double.doubleToLongBits: NaN canonicalised to 0x7ff8000000000000, as a signed long."""
    if math.isnan(d):
        return 0x7ff8000000000000
    return struct.unpack("<q", struct.pack("<d", d))[0]


def double_compare(a: float, b: float) -> int:
    """Double.compare (java.lang.Double:1000-1011)."""
    if a < b:
        return -1
    if a > b:
        return 1
    x, y = _double_to_long_bits(a), _double_to_long_bits(b)
    return 0 if x == y else (-1 if x < y else 1)


def value_compare(a, b, t: int) -> int:
    """NumberType.compare: NULL is the smallest value, two NULLs are equal."""
    if a is None and b is None:
        return 0
    if a is None:
        return -1
    if b is None:
        return 1
    if t == T_FP64:
        return double_compare(float(a), float(b))
    return (a > b) - (a < b)


def row_compare(x, y, types: Sequence[int], keys: Sequence[int], desc: Sequence[bool]) -> int:
    for k, d in zip(keys, desc):
        c = value_compare(x[k], y[k], types[k])
        if d:
            c = -c
        if c:
            return c
    return 0


def rows_of(cols) -> List[tuple]:
    n = len(cols[0][0]) if cols else 0
    out = []
    for r in range(n):
        row = []
        for v, nl in cols:
            if nl is not None and nl[r]:
                row.append(None)
            else:
                x = v[r]
                row.append(x.item() if hasattr(x, "item") else x)
        out.append(tuple(row))
    return out


def sort_rows(rows: Sequence[tuple], types: Sequence[int], keys: Sequence[int], desc: Sequence[bool],
              limit: Optional[int] = None) -> List[tuple]:
    out = sorted(rows, key=functools.cmp_to_key(lambda x, y: row_compare(x, y, types, keys, desc)))
    return out if limit is None else out[:limit]


# ------------------------------------------------------------------------------------------------ numpy form
def value_image(values: np.ndarray, t: int) -> np.ndarray:
    """uint64 whose unsigned order is the value order: integers with the sign bit flipped; doubles with NaN canonicalised,
    negatives complemented and the sign bit set on the rest."""
    if t == T_FP64:
        v = np.asarray(values, dtype=np.float64)
        b = v.view(np.uint64).copy()
        b[np.isnan(v)] = np.uint64(0x7ff8000000000000)
        neg = (b >> np.uint64(63)) == 1
        return np.where(neg, ~b, b | np.uint64(1 << 63))
    return np.asarray(values).astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63)


def key_columns(cols, types: Sequence[int], keys: Sequence[int], desc: Sequence[bool]) -> List[np.ndarray]:
    """Per key, most significant first: [non-NULL flag, image of the value (0 for NULL)], each complemented under DESC."""
    out = []
    for k, d in zip(keys, desc):
        v, nl = cols[k]
        isnull = np.zeros(len(v), bool) if nl is None else np.asarray(nl).astype(bool)
        flag = (~isnull).astype(np.uint64)
        img = np.where(isnull, np.uint64(0), value_image(v, types[k]))
        if d:
            flag, img = np.uint64(1) - flag, ~img
        out += [flag, img]
    return out


def lexsort_perm(cols, types, keys, desc) -> np.ndarray:
    ks = key_columns(cols, types, keys, desc)
    if not ks or len(ks[0]) == 0:
        return np.zeros(0, np.int64)
    return np.lexsort(ks[::-1])


def key_matrix(cols, types, keys, desc=None) -> np.ndarray:
    """(rows, 2 * nkeys) uint64: rows with equal keys under the comparator have equal lines (direction does not matter)."""
    ks = key_columns(cols, types, keys, [False] * len(keys))
    n = len(cols[0][0])
    return np.stack(ks, axis=1) if ks else np.zeros((n, 0), np.uint64)


def row_matrix(cols) -> np.ndarray:
    """(rows, 2 * ncols) int64 of (NULL flag, raw value bits, 0 under NULL): the exact identity of a row."""
    parts = []
    for v, nl in cols:
        v = np.asarray(v)
        isnull = np.zeros(len(v), bool) if nl is None else np.asarray(nl).astype(bool)
        bits = v.astype(np.int64) if v.dtype == np.int32 else v.view(np.int64)
        parts += [isnull.astype(np.int64), np.where(isnull, 0, bits)]
    return np.stack(parts, axis=1) if parts else np.zeros((0, 0), np.int64)


def _counter(m: np.ndarray) -> Counter:
    return Counter(map(bytes, np.ascontiguousarray(m)))


def check_ordered(out_cols, in_cols, types, keys, desc, limit: Optional[int] = None):
    """Asserts gsql_sort's contract on an output: its key sequence is the reference's exactly; its rows are a sub-multiset
    of the input (the input itself for a full sort); every input row strictly ahead of the last output key is present."""
    n_in = len(in_cols[0][0])
    n_out = len(out_cols[0][0])
    want = n_in if limit is None else min(limit, n_in)
    assert n_out == want, (n_out, want)
    perm = lexsort_perm(in_cols, types, keys, desc)
    ref_keys = key_matrix(in_cols, types, keys)[perm[:want]]
    got_keys = key_matrix(out_cols, types, keys)
    assert np.array_equal(got_keys, ref_keys), "key sequence differs from the comparator's order"
    rin, rout = row_matrix(in_cols), row_matrix(out_cols)
    cin, cout = _counter(rin), _counter(rout)
    if limit is None or want == n_in:
        assert cin == cout, "rows are not the input's multiset"
        return
    assert not (cout - cin), "output holds rows the input does not"
    if want == 0:
        return
    # rows strictly ahead of the last kept key: exactly the input's rows ranked before the first row with that key
    last = ref_keys[-1]
    all_keys = key_matrix(in_cols, types, keys)[perm]
    first_tie = int(np.argmax(np.all(all_keys == last, axis=1)))
    ahead_in = _counter(rin[perm[:first_tie]])
    ahead_out = _counter(rout[:first_tie])
    assert ahead_in == ahead_out, "a row strictly ahead of the boundary key is missing"
