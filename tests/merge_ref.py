"""The stable merge gsql_merge_* promises, restated over numpy columns for the merge tests: each input cut to its first
`limit` rows (the per-input quota), the inputs concatenated in index order, then a stable sort under the executor's
comparator (tests/sort_ref.py's lexsort form; numpy's lexsort is stable).  For inputs that are each ordered this is
exactly the stable k-way merge, row for row."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from tests import sort_ref as sr


def concat(inputs: Sequence[Sequence[tuple]], quota: Optional[int] = None) -> List[tuple]:
    """Columns of every input (each cut to `quota` rows) back to back; a NULL mask for every column."""
    ncols = len(inputs[0])
    out = []
    for c in range(ncols):
        ds, ns = [], []
        for cols in inputs:
            d, nl = cols[c]
            d = np.asarray(d)
            nl = np.zeros(len(d), bool) if nl is None else np.asarray(nl).astype(bool)
            if quota is not None:
                d, nl = d[:quota], nl[:quota]
            ds.append(d)
            ns.append(nl)
        out.append((np.concatenate(ds), np.concatenate(ns)))
    return out


def merged(inputs, types, keys, desc, limit: Optional[int] = None) -> List[tuple]:
    cat = concat(inputs, limit)
    perm = sr.lexsort_perm(cat, types, keys, desc)
    if limit is not None:
        perm = perm[:limit]
    return [(d[perm], nl[perm]) for d, nl in cat]


def of_rows(rows: Sequence[Sequence], types: Sequence[int]) -> List[tuple]:
    """Columns (values, nulls) of rows given as Python lists with None for NULL (one list per column)."""
    np_t = {sr.T_INT32: np.int32, sr.T_INT64: np.int64, sr.T_FP64: np.float64}
    return [(np.array([0 if v is None else v for v in col], dtype=np_t[t]), np.array([v is None for v in col], bool))
            for col, t in zip(rows, types)]


def assert_rows_equal(got, want):
    """Row for row: NULL flags and raw value bits."""
    a, b = sr.row_matrix(got), sr.row_matrix(want)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.array_equal(a, b), "rows differ from the stable merge"
