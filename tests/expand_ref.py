"""Restatement of ExpandExec + HashAggExec for tests (numpy only; nothing here runs on the GPU).

`expand` follows EX/operator/ExpandExec.java:48-69: every input chunk becomes one output chunk per projection, in
projection order, and projection s's output column c is the input column it references (same type and NULLs), a NULL,
or an integer constant.  `reference` aggregates that output with tests/agg_exact.Reference, grouped by the agg's group
columns (the set id `$e` among them), so its groups are exactly the stock operators' result as a multiset.

Projection items: an int (input column), None (NULL) or ("const", value), as api.GroupingSetsAgg takes them."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from tests import agg_exact as ax
from galaxysql_b200 import native as N

Col = Tuple[np.ndarray, Optional[np.ndarray]]
_NP = {N.T_INT32: np.int32, N.T_INT64: np.int64, N.T_FP64: np.float64}


def _item(cols: Sequence[Col], item, out_type: int, n: int, lo: int, hi: int) -> Col:
    if item is None:
        return np.zeros(n, _NP[out_type]), np.ones(n, bool)
    if isinstance(item, tuple):
        return np.full(n, item[1], _NP[out_type]), np.zeros(n, bool)
    d, nl = cols[item]
    assert np.asarray(d).dtype == _NP[out_type], "a reference keeps its column's type"
    return np.asarray(d)[lo:hi], (np.zeros(n, bool) if nl is None else np.asarray(nl, bool)[lo:hi])


def expand(cols: Sequence[Col], out_types: Sequence[int], projections, edges: Sequence[int]) -> List[Col]:
    """The Expand's output over input chunks [edges[i], edges[i+1]), concatenated in the order ExpandExec emits it."""
    parts: List[List[Col]] = []
    for lo, hi in zip(edges[:-1], edges[1:]):
        for proj in projections:
            parts.append([_item(cols, it, t, hi - lo, lo, hi) for it, t in zip(proj, out_types)])
    if not parts:
        return [(np.zeros(0, _NP[t]), np.zeros(0, bool)) for t in out_types]
    return [(np.concatenate([p[c][0] for p in parts]), np.concatenate([p[c][1] for p in parts])) for c in range(len(out_types))]


def reference(cols: Sequence[Col], out_types: Sequence[int], projections, groups: Sequence[int], aggs,
              filter_args: Optional[Sequence[int]] = None, edges: Optional[Sequence[int]] = None) -> ax.Reference:
    n = len(cols[0][0]) if cols else 0
    return ax.Reference(expand(cols, out_types, projections, edges if edges is not None else [0, n]), groups, aggs,
                        filter_args=filter_args)


# ------------------------------------------------------------------------------------------------ plan shapes
def rollup(keys: Sequence[int], values: Sequence[int]):
    """GroupingSetsToExpandRule's projections for ROLLUP(keys): output = keys..., values..., $e (BIGINT).  Set i keeps
    the first len(keys) - i keys."""
    nk = len(keys)
    return [[k if j < nk - i else None for j, k in enumerate(keys)] + list(values) + [("const", i)] for i in range(nk + 1)]


def cube(keys: Sequence[int], values: Sequence[int]):
    """CUBE(keys): one set per subset, the full set first (set id = bit mask of the dropped keys)."""
    nk = len(keys)
    return [[None if (m >> j) & 1 else k for j, k in enumerate(keys)] + list(values) + [("const", m)] for m in range(1 << nk)]


def grouping_sets(keys: Sequence[int], sets: Sequence[Sequence[int]], values: Sequence[int]):
    """GROUPING SETS over `keys`: sets[i] lists the positions (into keys) set i keeps."""
    return [[k if j in s else None for j, k in enumerate(keys)] + list(values) + [("const", i)] for i, s in enumerate(sets)]
