"""GPU-side helpers for the parity tests: run the C-ABI operators on (numpy | torch) columns and hand back numpy
columns shaped like the oracle's results."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from galaxysql_b200 import api, native as N
from oracle import oracle as orc  # the checker (tests only)

Col = Tuple[np.ndarray, Optional[np.ndarray]]

_CTX = None


def ctx() -> api.Context:
    global _CTX
    if _CTX is None:
        _CTX = api.Context(0)
    return _CTX


def _types(cols: Sequence[Col]) -> List[int]:
    m = {np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}
    return [m[np.asarray(d).dtype] for d, _ in cols]


def to_device(cols: Sequence[Col]):
    import torch
    out = []
    for d, nl in cols:
        td = torch.from_numpy(np.ascontiguousarray(d)).cuda()
        tn = None if nl is None else torch.from_numpy(np.ascontiguousarray(np.asarray(nl).astype(np.uint8))).cuda()
        out.append((td, tn))
    return out


def to_numpy(cols) -> List[Col]:
    out = []
    for d, nl in cols:
        if hasattr(d, "cpu"):
            d = d.cpu().numpy()
        if nl is not None and hasattr(nl, "cpu"):
            nl = nl.cpu().numpy()
        out.append((np.asarray(d), None if nl is None else np.asarray(nl).astype(bool)))
    return out


def _slice(cols, a, b):
    return [(d[a:b], None if nl is None else nl[a:b]) for d, nl in cols]


def _concat(parts: List[List[Col]]) -> List[Col]:
    if len(parts) == 1:
        return parts[0]
    out = []
    for c in range(len(parts[0])):
        d = np.concatenate([p[c][0] for p in parts])
        nl = np.concatenate([(p[c][1] if p[c][1] is not None else np.zeros(len(p[c][0]), bool)) for p in parts])
        out.append((d, nl))
    return out


def gpu_hash_join(spec: "orc.JoinSpec", outer: Sequence[Col], inner: Sequence[Col], mem: str = "host",
                  build_batches: int = 1, probe_batches: int = 1) -> List[Col]:
    """Same signature as oracle.hash_join, executed by libgsql_gpu.so."""
    c = ctx()
    j = api.HashJoin(c, spec.join_type, _types(outer), _types(inner), list(spec.outer_keys), list(spec.inner_keys),
                     list(spec.key_types), max_one_row=spec.max_one_row, build_outer=spec.build_outer,
                     anti_operands=spec.anti_operands, cond_ne=spec.cond_ne)
    build, probe = (outer, inner) if spec.build_outer else (inner, outer)
    nb = len(build[0][0])
    if nb:
        edges = np.linspace(0, nb, build_batches + 1).astype(int)
        for a, b in zip(edges[:-1], edges[1:]):
            part = _slice(build, a, b)
            j.build_consume(to_device(part) if mem == "device" else part)
    j.build_finish()
    npr = len(probe[0][0])
    parts = []
    edges = np.linspace(0, npr, probe_batches + 1).astype(int)
    for a, b in zip(edges[:-1], edges[1:]):
        part = _slice(probe, a, b)
        if b > a or probe_batches == 1:
            parts.append(to_numpy(j.probe(to_device(part) if mem == "device" else part)))
    if spec.build_outer:
        parts.append(to_numpy(j.unmatched_build(N.MEM_DEVICE if mem == "device" else N.MEM_HOST)))
    j.close()
    return _concat(parts)


_AGG_KIND = {orc.AGG_COUNT_STAR: N.AGG_COUNT_STAR, orc.AGG_COUNT: N.AGG_COUNT, orc.AGG_SUM: N.AGG_SUM,
             orc.AGG_AVG: N.AGG_AVG, orc.AGG_MIN: N.AGG_MIN, orc.AGG_MAX: N.AGG_MAX, orc.AGG_SUM0: N.AGG_SUM0}


def gpu_hash_agg(cols: Sequence[Col], groups: Sequence[int], aggs: Sequence["orc.AggCall"], expected_groups: int = 1024,
                 mem: str = "host", batches: int = 1) -> List[Col]:
    """Same signature as oracle.hash_agg.  DEC128 results come back as Python-int object arrays like the oracle's."""
    c = ctx()
    a = api.HashAgg(c, _types(cols), list(groups), [(_AGG_KIND[x.kind], list(x.cols)) for x in aggs], expected_groups,
                    filter_args=[x.filter_arg for x in aggs])
    n = len(cols[0][0]) if cols else 0
    edges = np.linspace(0, n, batches + 1).astype(int)
    for lo, hi in zip(edges[:-1], edges[1:]):
        part = _slice(cols, lo, hi)
        if hi > lo:
            a.consume(to_device(part) if mem == "device" else part)
    res = a.result(N.MEM_DEVICE if mem == "device" else N.MEM_HOST)
    out = []
    for (d, nl), t in zip(res, a.out_types):
        if hasattr(d, "cpu"):
            d, nl = d.cpu().numpy(), nl.cpu().numpy()
        if t == N.T_DEC128:
            d = np.array(api.dec128_to_int(d), dtype=object)
        out.append((np.asarray(d), np.asarray(nl).astype(bool)))
    a.close()
    return out


def gpu_partition(cols: Sequence[Col], channels: Sequence[int], nparts: int, mem: str = "host"):
    c = ctx()
    x = api.Exchange(c, _types(cols), list(channels), nparts)
    out, counts = x.partition(to_device(cols) if mem == "device" else cols)
    x.close()
    return to_numpy(out), counts


def approx_rows_equal(a: Sequence[Col], b: Sequence[Col], float_cols: Sequence[int], key_cols: Sequence[int], rtol=1e-6):
    """Sort both results by key columns; integer columns bit-exact, float columns within rtol.  Keys sort on their own
    values: integer keys beyond 2^53 would tie as float64.  (tests/agg_exact.py checks floating aggregates exactly.)"""
    def order(cols):
        keys = []
        for c in reversed(list(key_cols)):
            d, nl = cols[c]
            d = np.asarray(d)
            keys.append(d if d.dtype != object else d.astype(np.float64))
            keys.append(np.zeros(len(d), bool) if nl is None else np.asarray(nl, bool))
        return np.lexsort(keys) if keys else np.arange(len(cols[0][0]))
    assert len(a) == len(b)
    if len(a) == 0:
        return
    assert len(a[0][0]) == len(b[0][0]), (len(a[0][0]), len(b[0][0]))
    oa, ob = order(a), order(b)
    for c in range(len(a)):
        da, na = a[c]
        db, nb = b[c]
        na = np.zeros(len(da), bool) if na is None else np.asarray(na, bool)
        nb = np.zeros(len(db), bool) if nb is None else np.asarray(nb, bool)
        assert np.array_equal(na[oa], nb[ob]), f"null mask differs in column {c}"
        va, vb = np.asarray(da)[oa][~na[oa]], np.asarray(db)[ob][~nb[ob]]
        if c in float_cols:
            assert np.allclose(va.astype(np.float64), vb.astype(np.float64), rtol=rtol, atol=0), f"float column {c}"
        else:
            assert np.array_equal(va, vb), f"column {c} not bit-exact"
