"""Thin object layer over the C-ABI: Context, HashJoin, HashAgg, Exchange.

Columns are ``(values, nulls)`` pairs.  ``values`` is a numpy array (host batch) or a torch CUDA tensor
(device-resident batch); ``nulls`` is None or a uint8/bool array/tensor of the same length (non-zero = NULL) —
the Block convention of the reference (EX/chunk/AbstractBlock.java:27-47).  All columns of one call must live
in the same memory space.  Every compute call goes through libgsql_gpu.so; nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import native as N

try:  # torch is plumbing (device tensors, streams); the ABI itself does not need it
    import torch
except Exception:  # pragma: no cover
    torch = None

_NP_T = {np.dtype(np.int32): N.T_INT32, np.dtype(np.int64): N.T_INT64, np.dtype(np.float64): N.T_FP64}
_T_NP = {N.T_INT32: np.int32, N.T_INT64: np.int64, N.T_FP64: np.float64}


def _is_tensor(x) -> bool:
    return torch is not None and isinstance(x, torch.Tensor)


def _torch_t():
    return {torch.int32: N.T_INT32, torch.int64: N.T_INT64, torch.float64: N.T_FP64}


def _t_torch():
    return {N.T_INT32: torch.int32, N.T_INT64: torch.int64, N.T_FP64: torch.float64}


class _BatchView:
    """Builds a gsql_batch over numpy arrays or CUDA tensors and keeps them alive."""

    def __init__(self, cols: Sequence[Tuple[object, Optional[object]]], rows: Optional[int] = None):
        self.keep = []
        n = len(cols)
        self.carr = (N.Col * max(n, 1))()
        self.mem = N.MEM_HOST
        self.rows = 0 if rows is None else rows
        self.types = []
        for i, (data, nulls) in enumerate(cols):
            if _is_tensor(data):
                if not data.is_cuda:
                    raise TypeError("torch columns must be CUDA tensors (use numpy for host batches)")
                data = data.contiguous()
                self.mem = N.MEM_DEVICE
                t = _torch_t()[data.dtype]
                ptr = data.data_ptr()
                length = data.numel()
                nptr = 0
                if nulls is not None:
                    nulls = nulls.contiguous()
                    if nulls.dtype == torch.bool:
                        nulls = nulls.view(torch.uint8)
                    assert nulls.dtype == torch.uint8 and nulls.numel() == length
                    nptr = nulls.data_ptr()
                    self.keep.append(nulls)
            else:
                data = np.ascontiguousarray(data)
                if data.dtype not in _NP_T:
                    raise TypeError(f"unsupported dtype {data.dtype}")
                t = _NP_T[data.dtype]
                ptr = data.ctypes.data
                length = data.shape[0]
                nptr = 0
                if nulls is not None:
                    nulls = np.ascontiguousarray(np.asarray(nulls)).view(np.uint8) if np.asarray(nulls).dtype == np.bool_ \
                        else np.ascontiguousarray(nulls, dtype=np.uint8)
                    assert nulls.shape[0] == length
                    nptr = nulls.ctypes.data
                    self.keep.append(nulls)
            self.keep.append(data)
            self.carr[i].type = t
            self.carr[i].data = ptr
            self.carr[i].nulls = nptr
            self.types.append(t)
            if rows is None:
                self.rows = length
        self.batch = N.Batch(self.rows, n, self.mem, self.carr)

    def ref(self):
        return C.byref(self.batch)


class Context:
    """One GPU execution context (gsql_ctx): a device, a stream, an error slot."""

    def __init__(self, device: int = 0):
        self.lib = N.load()
        p = C.c_void_p()
        st = self.lib.gsql_ctx_create(device, C.byref(p))
        if st != N.OK:
            raise N.GsqlError(st, f"gsql_ctx_create(device={device}) failed: no usable CUDA device — "
                                  "galaxysql_b200 has no CPU fallback")
        self.ptr = p
        self.device = device
        self.nranks, self.rank = 1, 0   # set by comm_init

    def close(self):
        if getattr(self, "ptr", None):
            self.lib.gsql_ctx_destroy(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, st, required=None):
        N.check(self.ptr, st, required)

    def sync(self):
        self.check(self.lib.gsql_ctx_sync(self.ptr))

    @property
    def stream_ptr(self) -> int:
        return self.lib.gsql_ctx_stream(self.ptr) or 0

    def torch_stream(self):
        return torch.cuda.ExternalStream(self.stream_ptr, device=f"cuda:{self.device}")

    def set_stream(self, cuda_stream_ptr: int):
        self.check(self.lib.gsql_ctx_set_stream(self.ptr, C.c_void_p(cuda_stream_ptr)))

    def profile(self, enable: bool = True):
        self.check(self.lib.gsql_ctx_profile(self.ptr, int(enable)))

    def profile_reset(self):
        self.check(self.lib.gsql_ctx_profile_reset(self.ptr))

    def profile_get(self, name: str):
        n, ms = C.c_int64(), C.c_double()
        self.check(self.lib.gsql_ctx_profile_get(self.ptr, name.encode(), C.byref(n), C.byref(ms)))
        return n.value, ms.value

    def profile_dump(self):
        buf = C.create_string_buffer(1 << 16)
        self.lib.gsql_ctx_profile_dump(self.ptr, buf, len(buf))
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms = line.split()
            out[name] = (int(n), float(ms))
        return out

    @property
    def launch_count(self) -> int:
        return self.lib.gsql_ctx_launch_count(self.ptr)

    # ---- contractual hash utilities
    def hash_rows(self, cols, key_cols: Sequence[int], unified_types: Optional[Sequence[int]] = None):
        bv = _BatchView(cols)
        nk = len(key_cols)
        kc = (C.c_int32 * max(nk, 1))(*key_cols)
        ut = (C.c_int32 * max(nk, 1))(*(unified_types or [bv.types[c] for c in key_cols]))
        if bv.mem == N.MEM_DEVICE:
            out = torch.empty(bv.rows, dtype=torch.int32, device=f"cuda:{self.device}")
            optr = out.data_ptr()
        else:
            out = np.empty(bv.rows, dtype=np.int32)
            optr = out.ctypes.data
        self.check(self.lib.gsql_hash_rows(self.ptr, bv.ref(), kc, nk, ut, C.c_void_p(optr)))
        if bv.mem == N.MEM_DEVICE:
            self.sync()
        return out

    def partition_ids(self, hashes, nparts: int):
        if _is_tensor(hashes):
            out = torch.empty_like(hashes)
            self.check(self.lib.gsql_partition_ids(self.ptr, C.c_void_p(hashes.data_ptr()), hashes.numel(), nparts,
                                                   C.c_void_p(out.data_ptr()), N.MEM_DEVICE))
            self.sync()
            return out
        hashes = np.ascontiguousarray(hashes, dtype=np.int32)
        out = np.empty_like(hashes)
        self.check(self.lib.gsql_partition_ids(self.ptr, C.c_void_p(hashes.ctypes.data), hashes.size, nparts,
                                               C.c_void_p(out.ctypes.data), N.MEM_HOST))
        return out


def _alloc_out(ctx: Context, types: Sequence[int], rows: int, mem: int, with_nulls: Sequence[bool]):
    """Output columns for `rows` rows in the given memory space."""
    cols = []
    for t, wn in zip(types, with_nulls):
        if mem == N.MEM_DEVICE:
            dev = f"cuda:{ctx.device}"
            if t == N.T_DEC128:
                d = torch.empty((max(rows, 1), 2), dtype=torch.int64, device=dev)
            else:
                d = torch.empty(max(rows, 1), dtype=_t_torch()[t], device=dev)
            nl = torch.empty(max(rows, 1), dtype=torch.uint8, device=dev) if wn else None
        else:
            if t == N.T_DEC128:
                d = np.empty((max(rows, 1), 2), dtype=np.int64)
            else:
                d = np.empty(max(rows, 1), dtype=_T_NP[t])
            nl = np.empty(max(rows, 1), dtype=np.uint8) if wn else None
        cols.append((d, nl))
    return cols


def _out_batch(cols, types, rows, mem):
    n = len(cols)
    carr = (N.Col * max(n, 1))()
    for i, ((d, nl), t) in enumerate(zip(cols, types)):
        carr[i].type = t
        carr[i].data = d.data_ptr() if _is_tensor(d) else d.ctypes.data
        carr[i].nulls = 0 if nl is None else (nl.data_ptr() if _is_tensor(nl) else nl.ctypes.data)
    return N.Batch(rows, n, mem, carr), carr


def _trim(cols, rows):
    out = []
    for d, nl in cols:
        out.append((d[:rows], None if nl is None else nl[:rows]))
    return out


def dec128_to_int(col) -> List[int]:
    """DEC128 column ((rows,2) int64: lo, hi) -> Python ints."""
    a = col.cpu().numpy() if _is_tensor(col) else col
    lo = a[:, 0].astype(np.uint64)
    hi = a[:, 1]
    return [int(h) * (1 << 64) + int(l) for h, l in zip(hi.tolist(), lo.tolist())]


def _join_spec(join_type: int, outer_types: Sequence[int], inner_types: Sequence[int], outer_keys: Sequence[int],
               inner_keys: Sequence[int], key_types: Optional[Sequence[int]], max_one_row: bool, build_outer: bool,
               anti_operands: Optional[Sequence[int]], cond_ne: Sequence[Tuple[int, int]]) -> N.JoinSpec:
    s = N.JoinSpec()
    s.join_type, s.max_one_row, s.build_outer = join_type, int(max_one_row), int(build_outer)
    s.nkeys = len(outer_keys)
    key_types = key_types or [outer_types[k] for k in outer_keys]
    for i, (o, n_, t) in enumerate(zip(outer_keys, inner_keys, key_types)):
        s.outer_key[i], s.inner_key[i], s.key_type[i] = o, n_, t
    s.n_outer_cols = len(outer_types)
    for i, t in enumerate(outer_types):
        s.outer_types[i] = t
    s.n_inner_cols = len(inner_types)
    for i, t in enumerate(inner_types):
        s.inner_types[i] = t
    ops = list(anti_operands or [])
    s.n_anti_operands = len(ops)
    for i, o in enumerate(ops):
        s.anti_operands[i] = o
    s.n_cond = len(cond_ne)
    for i, (c, v) in enumerate(cond_ne):
        s.cond_col[i], s.cond_ne_value[i] = c, v
    return s


class HashJoin:
    """gsql_join handle: ParallelHashJoinExec's build + probe on the GPU."""

    def __init__(self, ctx: Context, join_type: int, outer_types: Sequence[int], inner_types: Sequence[int],
                 outer_keys: Sequence[int], inner_keys: Sequence[int], key_types: Optional[Sequence[int]] = None,
                 max_one_row: bool = False, build_outer: bool = False, anti_operands: Optional[Sequence[int]] = None,
                 cond_ne: Sequence[Tuple[int, int]] = (), expected_build_rows: int = 0):
        self.ctx = ctx
        s = _join_spec(join_type, outer_types, inner_types, outer_keys, inner_keys, key_types, max_one_row, build_outer,
                       anti_operands, cond_ne)
        s.expected_build_rows = expected_build_rows
        self.spec = s
        self.build_outer = build_outer
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_join_create(ctx.ptr, C.byref(s), C.byref(h)))
        self.h = h
        n = C.c_int32()
        types = (C.c_int32 * (2 * N.MAX_COLS))()
        ctx.check(ctx.lib.gsql_join_output_schema(self.h, C.byref(n), types))
        self.out_types = [types[i] for i in range(n.value)]

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_join_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def build_consume(self, cols):
        bv = _BatchView(cols)
        self.ctx.check(self.ctx.lib.gsql_join_build_consume(self.h, bv.ref()))

    def build_consume_ref(self, cols):
        """Zero-copy build side (one device-resident batch, e.g. the view an Exchange.recv returned): the columns are
        referenced until close()."""
        bv = _BatchView(cols)
        self._build_ref = bv  # keeps the tensors alive as long as the handle references them
        self.ctx.check(self.ctx.lib.gsql_join_build_consume_ref(self.h, bv.ref()))

    def build_finish(self):
        self.ctx.check(self.ctx.lib.gsql_join_build_finish(self.h))

    def info(self) -> N.JoinInfo:
        i = N.JoinInfo()
        self.ctx.check(self.ctx.lib.gsql_join_info_get(self.h, C.byref(i)))
        return i

    def probe_count(self, cols) -> int:
        bv = _BatchView(cols)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_join_probe_count(self.h, bv.ref(), C.byref(n)))
        return n.value

    def probe_into(self, cols, out_cols, capacity: int) -> int:
        """Probe with caller-owned output columns (device-resident pipelines, bench)."""
        bv = _BatchView(cols)
        ob, _keep = _out_batch(out_cols, self.out_types, 0, bv.mem)
        n = C.c_int64()
        st = self.ctx.lib.gsql_join_probe(self.h, bv.ref(), C.byref(ob), capacity, C.byref(n))
        self.ctx.check(st, n.value)
        return n.value

    def probe(self, cols, capacity: Optional[int] = None, nullable_out: bool = True):
        """nextChunk over a probe batch -> list of (values, nulls) output columns."""
        bv = _BatchView(cols)
        cap = capacity if capacity is not None else max(bv.rows, 1)
        while True:
            out = _alloc_out(self.ctx, self.out_types, cap, bv.mem, [nullable_out] * len(self.out_types))
            ob, _keep = _out_batch(out, self.out_types, 0, bv.mem)
            n = C.c_int64()
            st = self.ctx.lib.gsql_join_probe(self.h, bv.ref(), C.byref(ob), cap, C.byref(n))
            if st == N.E_CAPACITY:
                cap = n.value
                continue
            self.ctx.check(st)
            if bv.mem == N.MEM_DEVICE:
                self.ctx.sync()
            return _trim(out, n.value)

    def unmatched_build(self, mem: int = N.MEM_HOST):
        cap = 1024
        while True:
            out = _alloc_out(self.ctx, self.out_types, cap, mem, [True] * len(self.out_types))
            ob, _keep = _out_batch(out, self.out_types, 0, mem)
            n = C.c_int64()
            st = self.ctx.lib.gsql_join_unmatched_build(self.h, C.byref(ob), cap, C.byref(n))
            if st == N.E_CAPACITY:
                cap = n.value
                continue
            self.ctx.check(st)
            if mem == N.MEM_DEVICE:
                self.ctx.sync()
            return _trim(out, n.value)


def _agg_spec(input_types: Sequence[int], groups: Sequence[int], aggs: Sequence[Tuple[int, Sequence[int]]],
              expected_groups: int, filter_args: Optional[Sequence[int]], derived: Sequence[Tuple[int, int, int, int]],
              row_filter: Optional[Tuple[int, int, int]]) -> N.AggSpec:
    s = N.AggSpec()
    s.n_input_cols = len(input_types)
    for i, t in enumerate(input_types):
        s.input_types[i] = t
    s.ngroups = len(groups)
    for i, g in enumerate(groups):
        s.groups[i] = g
    s.naggs = len(aggs)
    for i, (kind, cols) in enumerate(aggs):
        s.aggs[i].kind = kind
        s.aggs[i].ncols = len(cols)
        for k, c in enumerate(cols):
            s.aggs[i].cols[k] = c
        s.aggs[i].filter_arg = filter_args[i] if filter_args else -1
    s.expected_groups = expected_groups
    s.n_derived = len(derived)
    for i, (kind, a_, b_, c_) in enumerate(derived):
        s.derived[i].kind, s.derived[i].a, s.derived[i].b, s.derived[i].c = kind, a_, b_, c_
    if row_filter is not None:
        s.row_filter_col, s.row_filter_op, s.row_filter_value = row_filter
    else:
        s.row_filter_col, s.row_filter_op = -1, N.CMP_NONE
    return s


class HashAgg:
    """gsql_agg handle: HashAggExec's consume / buildConsume / nextChunk on the GPU."""

    def __init__(self, ctx: Context, input_types: Sequence[int], groups: Sequence[int],
                 aggs: Sequence[Tuple[int, Sequence[int]]], expected_groups: int = 1024,
                 filter_args: Optional[Sequence[int]] = None,
                 derived: Sequence[Tuple[int, int, int, int]] = (), row_filter: Optional[Tuple[int, int, int]] = None):
        """derived: (kind, a, b, c) fused FP64 expressions addressed as columns len(input_types)+i;
        row_filter: (column, gsql_cmp_op, value) fused scan-side predicate."""
        self.ctx = ctx
        s = _agg_spec(input_types, groups, aggs, expected_groups, filter_args, derived, row_filter)
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_agg_create(ctx.ptr, C.byref(s), C.byref(h)))
        self.h = h
        n = C.c_int32()
        types = (C.c_int32 * N.MAX_COLS)()
        ctx.check(ctx.lib.gsql_agg_output_schema(self.h, C.byref(n), types))
        self.out_types = [types[i] for i in range(n.value)]

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_agg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def consume(self, cols, rows: Optional[int] = None):
        bv = _BatchView(cols, rows)
        self.ctx.check(self.ctx.lib.gsql_agg_consume(self.h, bv.ref()))

    def finish(self) -> int:
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_agg_finish(self.h, C.byref(n)))
        return n.value

    def next(self, max_rows: int, mem: int = N.MEM_HOST):
        out = _alloc_out(self.ctx, self.out_types, max_rows, mem, [True] * len(self.out_types))
        ob, _keep = _out_batch(out, self.out_types, 0, mem)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_agg_next(self.h, C.byref(ob), max_rows, C.byref(n)))
        if mem == N.MEM_DEVICE:
            self.ctx.sync()
        return _trim(out, n.value)

    def result(self, mem: int = N.MEM_HOST):
        """finish() + drain everything."""
        n = self.finish()
        return self.next(max(n, 1), mem) if n > 0 else _trim(
            _alloc_out(self.ctx, self.out_types, 1, mem, [True] * len(self.out_types)), 0)


def _expand_spec(input_types: Sequence[int], output_types: Sequence[int], projections) -> N.ExpandSpec:
    e = N.ExpandSpec()
    e.n_input_cols = len(input_types)
    for i, t in enumerate(input_types):
        e.input_types[i] = t
    e.nsets, e.n_output_cols = len(projections), len(output_types)
    for s, proj in enumerate(projections[:N.MAX_SETS]):
        for c, item in enumerate(proj):
            it = e.proj[s][c]
            if item is None:
                it.src = N.EXPAND_NULL
            elif isinstance(item, tuple):
                it.src, it.value = N.EXPAND_CONST, item[1]
            else:
                it.src, it.col = N.EXPAND_INPUT, item
    return e


class GroupingSetsAgg(HashAgg):
    """gsql_gsagg handle: HashAggExec over ExpandExec (ROLLUP / CUBE / GROUPING SETS, DISTINCT rewrites) on the GPU, without
    materialising the Expand.  projections[s][c] is projection s's output column c: an int (that input column), None (NULL)
    or ("const", value).  output_types are the Expand's output types; groups, aggs and filter_args address its output
    columns, as HashAgg's do its input.  consume() takes the Expand's input; result() lists the sets in Expand order."""

    def __init__(self, ctx: Context, input_types: Sequence[int], output_types: Sequence[int], projections,
                 groups: Sequence[int], aggs: Sequence[Tuple[int, Sequence[int]]], expected_groups: int = 1024,
                 filter_args: Optional[Sequence[int]] = None,
                 derived: Sequence[Tuple[int, int, int, int]] = (), row_filter: Optional[Tuple[int, int, int]] = None):
        """derived and row_filter exist so that the library's refusal of them can be seen (GSQL_E_UNSUPPORTED)."""
        self.ctx = ctx
        e = _expand_spec(input_types, output_types, projections)
        s = _agg_spec(output_types, groups, aggs, expected_groups, filter_args, derived, row_filter)
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_gsagg_create(ctx.ptr, C.byref(e), C.byref(s), C.byref(h)))
        self.h = h
        n = C.c_int32()
        types = (C.c_int32 * N.MAX_COLS)()
        ctx.check(ctx.lib.gsql_gsagg_output_schema(self.h, C.byref(n), types))
        self.out_types = [types[i] for i in range(n.value)]

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_gsagg_destroy(self.h)
            self.h = None

    def consume(self, cols, rows: Optional[int] = None):
        bv = _BatchView(cols, rows)
        self.ctx.check(self.ctx.lib.gsql_gsagg_consume(self.h, bv.ref()))

    def finish(self) -> int:
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_gsagg_finish(self.h, C.byref(n)))
        return n.value

    def next(self, max_rows: int, mem: int = N.MEM_HOST):
        out = _alloc_out(self.ctx, self.out_types, max_rows, mem, [True] * len(self.out_types))
        ob, _keep = _out_batch(out, self.out_types, 0, mem)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_gsagg_next(self.h, C.byref(ob), max_rows, C.byref(n)))
        if mem == N.MEM_DEVICE:
            self.ctx.sync()
        return _trim(out, n.value)


class SortAgg:
    """gsql_sortagg handle: SortAggExec on the GPU.  One output row per run of adjacent rows with equal group keys, in input
    order; groups complete after a consume can be returned (next) while input is still arriving."""

    def __init__(self, ctx: Context, input_types: Sequence[int], groups: Sequence[int],
                 aggs: Sequence[Tuple[int, Sequence[int]]], filter_args: Optional[Sequence[int]] = None,
                 derived: Sequence[Tuple[int, int, int, int]] = (), row_filter: Optional[Tuple[int, int, int]] = None):
        """filter_args, derived and row_filter exist so that the library's refusal of them can be seen: any of them makes
        the constructor raise GsqlError (GSQL_E_UNSUPPORTED)."""
        self.ctx = ctx
        s = _agg_spec(input_types, groups, aggs, 0, filter_args, derived, row_filter)
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_sortagg_create(ctx.ptr, C.byref(s), C.byref(h)))
        self.h = h
        n = C.c_int32()
        types = (C.c_int32 * N.MAX_COLS)()
        ctx.check(ctx.lib.gsql_sortagg_output_schema(self.h, C.byref(n), types))
        self.out_types = [types[i] for i in range(n.value)]

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_sortagg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def consume(self, cols, rows: Optional[int] = None) -> int:
        """-> groups ready to be returned (complete and not yet returned)."""
        bv = _BatchView(cols, rows)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_sortagg_consume(self.h, bv.ref(), C.byref(n)))
        return n.value

    def finish(self) -> int:
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_sortagg_finish(self.h, C.byref(n)))
        return n.value

    def next(self, max_rows: int, mem: int = N.MEM_HOST, nullable_out: bool = True):
        out = _alloc_out(self.ctx, self.out_types, max_rows, mem, [nullable_out] * len(self.out_types))
        ob, _keep = _out_batch(out, self.out_types, 0, mem)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_sortagg_next(self.h, C.byref(ob), max_rows, C.byref(n)))
        if mem == N.MEM_DEVICE:
            self.ctx.sync()
        return _trim(out, n.value)

    def result(self, mem: int = N.MEM_HOST):
        """finish() + drain every ready group."""
        n = self.finish()
        return self.next(max(n, 1), mem)


class Window:
    """gsql_window handle: NonFrameOverWindowExec on the GPU.  Every call is a running value from the start of the row's
    partition to the row (ROW_NUMBER, RANK, DENSE_RANK, COUNT / SUM / SUM0 / AVG / MIN / MAX), written to every row; each
    batch continues the previous batch's last partition."""

    def __init__(self, ctx: Context, input_types: Sequence[int], partition: Sequence[int],
                 calls: Sequence[Tuple[int, Sequence[int]]], reset_each_row: bool = False,
                 filter_args: Optional[Sequence[int]] = None):
        """calls: (kind, columns) with kind an N.AGG_* value; RANK / DENSE_RANK take their peer (ORDER BY) columns.
        reset_each_row: the ROWS CURRENT ROW .. CURRENT ROW frame.  filter_args exists so that the library's refusal of
        FILTER can be seen: any value >= 0 makes the constructor raise GsqlError (GSQL_E_UNSUPPORTED)."""
        self.ctx = ctx
        s = N.WindowSpec()
        s.n_input_cols = len(input_types)
        for i, t in enumerate(input_types):
            s.input_types[i] = t
        s.npart = len(partition)
        for i, c in enumerate(partition):
            s.part_cols[i] = c
        s.ncalls = len(calls)
        for i, (kind, cols) in enumerate(calls):
            s.calls[i].kind = kind
            s.calls[i].ncols = len(cols)
            for k, c in enumerate(cols):
                s.calls[i].cols[k] = c
            s.calls[i].filter_arg = filter_args[i] if filter_args else -1
        s.reset_each_row = int(reset_each_row)
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_window_create(ctx.ptr, C.byref(s), C.byref(h)))
        self.h = h
        n = C.c_int32()
        types = (C.c_int32 * (N.MAX_COLS + N.MAX_AGGS))()
        ctx.check(ctx.lib.gsql_window_output_schema(self.h, C.byref(n), types))
        self.types = [types[i] for i in range(n.value)]  # the operator's schema: the inputs, then one column per call
        self.out_types = self.types[len(input_types):]

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_window_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def apply(self, cols, rows: Optional[int] = None, mem: Optional[int] = None, out_cols=None):
        """-> the call columns for the batch's rows ((values, nulls) each; DEC128 as (rows, 2) int64), in `mem` (default:
        the input's memory space).  The input columns themselves are the operator's leading output columns."""
        bv = _BatchView(cols, rows)
        mem = bv.mem if mem is None else mem
        out = out_cols if out_cols is not None else _alloc_out(self.ctx, self.out_types, max(bv.rows, 1), mem,
                                                                  [True] * len(self.out_types))
        ob, _keep = _out_batch(out, self.out_types, 0, mem)
        self.ctx.check(self.ctx.lib.gsql_window_apply(self.h, bv.ref(), C.byref(ob)))
        if mem == N.MEM_DEVICE:
            self.ctx.sync()
        return _trim(out, bv.rows)


class SortMergeJoin:
    """gsql_smj handle: SortMergeJoinExec on the GPU.  Both inputs are ordered on the join keys (desc[k]: key k is
    DESCENDING); rows come out in the stock operator's order.  The inner side is consumed whole, then each outer batch is
    probed and its rows drained with next() before the next probe."""

    def __init__(self, ctx: Context, join_type: int, outer_types: Sequence[int], inner_types: Sequence[int],
                 outer_keys: Sequence[int], inner_keys: Sequence[int], key_types: Optional[Sequence[int]] = None,
                 desc: Optional[Sequence[bool]] = None, max_one_row: bool = False,
                 anti_operands: Optional[Sequence[int]] = None, build_outer: bool = False,
                 cond_ne: Sequence[Tuple[int, int]] = ()):
        """build_outer and cond_ne exist so that the library's refusal of them can be seen: either makes the constructor
        raise GsqlError (GSQL_E_UNSUPPORTED)."""
        self.ctx = ctx
        s = _join_spec(join_type, outer_types, inner_types, outer_keys, inner_keys, key_types, max_one_row, build_outer,
                       anti_operands, cond_ne)
        nk = len(outer_keys)
        kd = (C.c_int32 * max(nk, 1))(*[int(bool(d)) for d in (desc or [False] * nk)])
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_smj_create(ctx.ptr, C.byref(s), kd, C.byref(h)))
        self.h = h
        n = C.c_int32()
        types = (C.c_int32 * (2 * N.MAX_COLS))()
        ctx.check(ctx.lib.gsql_smj_output_schema(self.h, C.byref(n), types))
        self.out_types = [types[i] for i in range(n.value)]
        self._outer = None

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_smj_destroy(self.h)
            self.h = None
        self._outer = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def inner_consume(self, cols):
        bv = _BatchView(cols)
        self.ctx.check(self.ctx.lib.gsql_smj_inner_consume(self.h, bv.ref()))

    def inner_finish(self):
        self.ctx.check(self.ctx.lib.gsql_smj_inner_finish(self.h))

    def probe(self, cols) -> int:
        """-> the exact number of rows next() returns for this outer batch.  A device batch is referenced until next()
        returns 0 rows, so its tensors are kept alive here until then."""
        bv = _BatchView(cols)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_smj_probe(self.h, bv.ref(), C.byref(n)))
        self._outer = bv
        return n.value

    def next(self, max_rows: int, mem: int = N.MEM_HOST, nullable_out: bool = True):
        out = _alloc_out(self.ctx, self.out_types, max_rows, mem, [nullable_out] * len(self.out_types))
        ob, _keep = _out_batch(out, self.out_types, 0, mem)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_smj_next(self.h, C.byref(ob), max_rows, C.byref(n)))
        if mem == N.MEM_DEVICE:
            self.ctx.sync()
        if n.value == 0:
            self._outer = None
        return _trim(out, n.value)

    def join(self, cols, mem: int = N.MEM_HOST):
        """probe() + every row of the batch in one call (and the closing next() that releases it)."""
        n = self.probe(cols)
        out = self.next(max(n, 1), mem)
        self.next(1, mem)
        return out


class E:
    """Expression builder for Scan: E.col(i), E.lit(v) and Python operators -> a postfix program (gsql_expr).
    `&`, `|`, `~` are SQL AND / OR / NOT; comparisons yield BIGINT 0/1; `/` is DOUBLE division, NULL where the divisor is
    zero; to_i64() of a double rounds half to even and saturates (CAST ... AS SIGNED), NaN -> 0."""

    def __init__(self, ins):
        self.ins = ins  # list of (op, arg, const)

    @staticmethod
    def col(i: int) -> "E":
        return E([(N.OP_COL, i, 0)])

    @staticmethod
    def lit(v) -> "E":
        if isinstance(v, float):
            return E([(N.OP_CONST_F64, 0, float(v))])
        return E([(N.OP_CONST_I64, 0, int(v))])

    @staticmethod
    def _wrap(v) -> "E":
        return v if isinstance(v, E) else E.lit(v)

    def _bin(self, other, op, swap=False):
        o = E._wrap(other)
        a, b = (o, self) if swap else (self, o)
        return E(a.ins + b.ins + [(op, 0, 0)])

    def __add__(self, o): return self._bin(o, N.OP_ADD)
    def __radd__(self, o): return self._bin(o, N.OP_ADD, True)
    def __sub__(self, o): return self._bin(o, N.OP_SUB)
    def __rsub__(self, o): return self._bin(o, N.OP_SUB, True)
    def __mul__(self, o): return self._bin(o, N.OP_MUL)
    def __rmul__(self, o): return self._bin(o, N.OP_MUL, True)
    def __truediv__(self, o): return self._bin(o, N.OP_DIV)
    def __rtruediv__(self, o): return self._bin(o, N.OP_DIV, True)
    def __lt__(self, o): return self._bin(o, N.OP_LT)
    def __le__(self, o): return self._bin(o, N.OP_LE)
    def __gt__(self, o): return self._bin(o, N.OP_GT)
    def __ge__(self, o): return self._bin(o, N.OP_GE)
    def eq(self, o): return self._bin(o, N.OP_EQ)
    def ne(self, o): return self._bin(o, N.OP_NE)
    def __and__(self, o): return self._bin(o, N.OP_AND)
    def __or__(self, o): return self._bin(o, N.OP_OR)
    def __invert__(self): return E(self.ins + [(N.OP_NOT, 0, 0)])
    def __neg__(self): return E(self.ins + [(N.OP_NEG, 0, 0)])
    def is_null(self): return E(self.ins + [(N.OP_IS_NULL, 0, 0)])
    def to_f64(self): return E(self.ins + [(N.OP_CAST_F64, 0, 0)])
    def to_i64(self): return E(self.ins + [(N.OP_CAST_I64, 0, 0)])

    # The conditional and set builders below make programs that only gsql_scan_create2 accepts; Scan picks it for them.
    # IN and BETWEEN carry their constants in the instruction as a tuple; Scan moves them into the constant pool.
    @staticmethod
    def null(type_: int) -> "E":
        """A NULL of type T_INT64 or T_FP64."""
        return E([(N.OP_CONST_NULL, type_, 0)])

    @staticmethod
    def case(*args, else_type: Optional[int] = None) -> "E":
        """case(c1, v1, c2, v2, ..., [else]): the value of the first TRUE condition (NULL and 0 are not TRUE), else the
        last argument; without one, NULL of `else_type` (T_INT64 or T_FP64, the type of the values).  Compiled right to
        left: else, cn, vn, CASE_WHEN, ..., c1, v1, CASE_WHEN."""
        args = [E._wrap(a) for a in args]
        if len(args) < 2:
            raise ValueError("case needs a condition and a value")
        if len(args) % 2 == 0:
            if else_type is None:
                raise ValueError("case without an else needs else_type")
            args.append(E.null(else_type))
        ins = args[-1].ins
        for i in range(len(args) - 3, -1, -2):
            ins = ins + args[i].ins + args[i + 1].ins + [(N.OP_CASE_WHEN, 0, 0)]
        return E(ins)

    @staticmethod
    def coalesce(*args) -> "E":
        """The first argument that is not NULL; NULL if all are."""
        args = [E._wrap(a) for a in args]
        ins = args[0].ins
        for a in args[1:]:
            ins = ins + a.ins + [(N.OP_COALESCE, 0, 0)]
        return E(ins)

    def isin(self, values) -> "E":
        """self IN (values), over an integer operand: never NULL; a NULL operand compares as 0 (see GSQL_OP_IN)."""
        return E(self.ins + [(N.OP_IN, 0, tuple(int(v) for v in values))])

    def between(self, lo, hi) -> "E":
        """lo <= self <= hi over an integer operand, with IN's NULL rule (GSQL_OP_BETWEEN)."""
        return E(self.ins + [(N.OP_BETWEEN, 0, (int(lo), int(hi)))])

    def has_pool_ops(self) -> bool:
        return any(op >= N.OP_CONST_NULL for op, _, _ in self.ins)

    def fill(self, dst: "N.Expr", pool: Optional[list] = None):
        """pool: the scan's constant pool, to which IN lists and BETWEEN bounds are appended."""
        if len(self.ins) > N.MAX_EXPR_INS:
            raise ValueError("expression too long")
        dst.n = len(self.ins)
        for i, (op, arg, k) in enumerate(self.ins):
            if op in (N.OP_IN, N.OP_BETWEEN):
                arg, k, consts = len(pool), len(k), k
                pool.extend(consts)
            dst.ins[i].op, dst.ins[i].arg = op, arg
            if op == N.OP_CONST_F64:
                dst.ins[i].k.d = k
            else:
                dst.ins[i].k.i = k


class Scan:
    """gsql_scan handle: vectorised Filter + Project in one pass (VectorizedFilterExec / VectorizedProjectExec)."""

    def __init__(self, ctx: Context, input_types: Sequence[int], outputs: Sequence["E"], filter: Optional["E"] = None):
        self.ctx = ctx
        s = N.ScanSpec()
        s.n_input_cols = len(input_types)
        for i, t in enumerate(input_types):
            s.input_types[i] = t
        s.has_filter = int(filter is not None)
        pool: List[int] = []
        if filter is not None:
            filter.fill(s.filter, pool)
        s.n_out = len(outputs)
        for i, e in enumerate(outputs):
            E._wrap(e).fill(s.out[i], pool)
        h = C.c_void_p()
        if any(E._wrap(e).has_pool_ops() for e in list(outputs) + ([filter] if filter is not None else [])):
            arr = (C.c_int64 * max(len(pool), 1))(*pool)
            ctx.check(ctx.lib.gsql_scan_create2(ctx.ptr, C.byref(s), arr, len(pool), C.byref(h)))
        else:
            ctx.check(ctx.lib.gsql_scan_create(ctx.ptr, C.byref(s), C.byref(h)))
        self.h = h
        n = C.c_int32()
        types = (C.c_int32 * N.MAX_SCAN_OUT)()
        ctx.check(ctx.lib.gsql_scan_output_schema(self.h, C.byref(n), types))
        self.out_types = [types[i] for i in range(n.value)]

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_scan_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def apply(self, cols, nullable_out: bool = True, out_cols=None):
        """-> surviving rows as (values, nulls) columns in the input's memory space (trimmed views of out_cols)."""
        bv = _BatchView(cols)
        cap = max(bv.rows, 1)
        out = out_cols if out_cols is not None else _alloc_out(self.ctx, self.out_types, cap, bv.mem, [nullable_out] * len(self.out_types))
        ob, _keep = _out_batch(out, self.out_types, 0, bv.mem)
        n = C.c_int64()
        st = self.ctx.lib.gsql_scan_apply(self.h, bv.ref(), C.byref(ob), cap if out_cols is None else int(out[0][0].shape[0]), C.byref(n))
        self.ctx.check(st, n.value)
        return _trim(out, n.value)


class Exchange:
    """gsql_xchg handle: hash-partition exchange (local partition, or partition-and-push across ranks)."""

    def __init__(self, ctx: Context, types: Sequence[int], channels: Sequence[int], nparts: int,
                 key_types: Optional[Sequence[int]] = None, mode: int = 0):
        self.ctx = ctx
        s = N.XchgSpec()
        s.mode = mode
        s.n_cols = len(types)
        for i, t in enumerate(types):
            s.types[i] = t
        s.n_channels = len(channels)
        kt = key_types or [types[c] for c in channels]
        for i, (c, t) in enumerate(zip(channels, kt)):
            s.channels[i], s.key_types[i] = c, t
        s.nparts = nparts
        self.types = list(types)
        self.nparts = nparts
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_xchg_create(ctx.ptr, C.byref(s), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_xchg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def partition(self, cols):
        bv = _BatchView(cols)
        wn = [nl is not None for _, nl in cols]
        out = _alloc_out(self.ctx, self.types, bv.rows, bv.mem, wn)
        ob, _keep = _out_batch(out, self.types, bv.rows, bv.mem)
        counts = (C.c_int64 * self.nparts)()
        self.ctx.check(self.ctx.lib.gsql_xchg_partition(self.h, bv.ref(), C.byref(ob), counts))
        if bv.mem == N.MEM_DEVICE:
            self.ctx.sync()
        return _trim(out, bv.rows), np.array(list(counts), dtype=np.int64)


class _DevView:
    """A typed window onto device memory the library owns (__cuda_array_interface__), so that torch can wrap it without a copy."""

    def __init__(self, ptr: int, n: int, typestr: str, owner):
        self.owner = owner
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


_TYPESTR = {N.T_INT32: "<i4", N.T_INT64: "<i8", N.T_FP64: "<f8"}


def _view_tensor(ctx: Context, ptr: int, n: int, t: Optional[int], owner):
    dev = f"cuda:{ctx.device}"
    if n == 0 or not ptr:
        return torch.empty(0, dtype=torch.uint8 if t is None else _t_torch()[t], device=dev)
    return torch.as_tensor(_DevView(ptr, n, "|u1" if t is None else _TYPESTR[t], owner), device=dev)


def _exchange_open_p2p(self, capacity_rows: int, nullable: Sequence[int] = ()):
    """Collective: allocate this rank's receive buffer (capacity_rows rows; the same value on every rank) and map every
    peer's buffer (gsql_xchg_open_p2p)."""
    mask = 0
    for c in nullable:
        mask |= 1 << c
    self.ctx.check(self.ctx.lib.gsql_xchg_open_p2p(self.h, capacity_rows, mask))
    self._nullable = set(nullable)


def _exchange_push(self, cols, nslabs: int = 1):
    """Collective, asynchronous: split `cols` (device) by destination rank and write every destination's rows straight
    into its receive buffer over NVLink, slab after slab.  Returns the rows this rank receives per slab."""
    bv = _BatchView(cols)
    assert bv.mem == N.MEM_DEVICE
    self._push_src = bv  # the input must stay alive until the slabs have been received
    rows = (C.c_int64 * nslabs)()
    total = C.c_int64()
    st = self.ctx.lib.gsql_xchg_push(self.h, bv.ref(), nslabs, rows, C.byref(total))
    self.ctx.check(st, total.value)
    return [rows[i] for i in range(nslabs)]


def _exchange_recv(self, slab: int = -1):
    """The rows of slab `slab` of the last push (-1: all slabs as one batch) as zero-copy tensors over the receive
    buffer; the context stream is made to wait for their arrival.  Valid until the next push."""
    n = len(self.types)
    carr = (N.Col * n)()
    view = N.Batch(0, n, N.MEM_DEVICE, carr)
    self.ctx.check(self.ctx.lib.gsql_xchg_recv_view(self.h, slab, C.byref(view)))
    out = []
    for c in range(n):
        d = _view_tensor(self.ctx, carr[c].data or 0, view.rows, self.types[c], self)
        nl = _view_tensor(self.ctx, carr[c].nulls or 0, view.rows, None, self) if carr[c].nulls else None
        out.append((d, nl))
    return out


def _exchange_push_wait(self):
    self.ctx.check(self.ctx.lib.gsql_xchg_push_wait(self.h))


Exchange.open_p2p = _exchange_open_p2p
Exchange.push = _exchange_push
Exchange.recv = _exchange_recv
Exchange.push_wait = _exchange_push_wait


def plan_layout(nranks: int, nslabs: int, me: int, matrix):
    """gsql_xchg_plan_layout (pure host arithmetic): matrix[src][slab][dst] -> (send_base[slab][dst], recv_base[slab][src],
    slab_rows[slab], worst rank's total)."""
    m = np.ascontiguousarray(matrix, dtype=np.int64).reshape(nranks, nslabs, nranks)
    send = np.zeros((nslabs, nranks), dtype=np.int64)
    recv = np.zeros((nslabs, nranks), dtype=np.int64)
    rows = np.zeros(nslabs, dtype=np.int64)
    p64 = C.POINTER(C.c_int64)
    worst = N.load().gsql_xchg_plan_layout(nranks, nslabs, me, m.ctypes.data_as(p64), send.ctypes.data_as(p64),
                                           recv.ctypes.data_as(p64), rows.ctypes.data_as(p64))
    return send, recv, rows, int(worst)


def serde_serialize(ctx: Context, cols, page_rows: int = 1024):
    """Chunk columns -> the reference's MPP wire bytes (gsql_serde_serialize): numpy uint8 for host columns, a CUDA uint8
    tensor for device columns."""
    bv = _BatchView(cols)
    need = C.c_int64()
    ctx.check(ctx.lib.gsql_serde_size(ctx.ptr, bv.ref(), page_rows, C.byref(need)))
    n = need.value
    if bv.mem == N.MEM_DEVICE:
        out = torch.empty(max(n, 1), dtype=torch.uint8, device=f"cuda:{ctx.device}")
        ptr = out.data_ptr()
    else:
        out = np.empty(max(n, 1), dtype=np.uint8)
        ptr = out.ctypes.data
    got = C.c_int64()
    ctx.check(ctx.lib.gsql_serde_serialize(ctx.ptr, bv.ref(), page_rows, C.c_void_p(ptr), n, C.byref(got)))
    assert got.value == n
    return out[:n]


def serde_deserialize(ctx: Context, data, types: Sequence[int]):
    """Wire bytes (numpy uint8 / bytes, or a CUDA uint8 tensor) -> [(values, nulls)] in the same memory space."""
    if _is_tensor(data):
        mem, ptr, nbytes = N.MEM_DEVICE, data.data_ptr(), data.numel()
    else:
        data = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data, dtype=np.uint8)
        mem, ptr, nbytes = N.MEM_HOST, data.ctypes.data, data.size
    cap = 0
    while True:
        out = _alloc_out(ctx, types, max(cap, 1), mem, [True] * len(types))
        ob, _keep = _out_batch(out, types, 0, mem)
        n = C.c_int64()
        st = ctx.lib.gsql_serde_deserialize(ctx.ptr, C.c_void_p(ptr), nbytes, mem, C.byref(ob), cap, C.byref(n))
        if st == N.E_CAPACITY:
            cap = n.value
            continue
        ctx.check(st)
        return _trim(out, n.value)


def bloom_sizing(ndv: int, min_size: int = 1000, max_size: int = 2 << 20) -> Tuple[int, int]:
    """(num_bits, num_hash_functions) of the runtime filter the reference's factory creates for a build side of `ndv`
    distinct keys (RuntimeFilterBuilderExecFactory.java:75-98): size = clamp(ndv, BLOOM_FILTER_MIN_SIZE, BLOOM_FILTER_MAX_SIZE),
    fpp = max(exp(-3.843 size / ndv), BloomFilter.DEFAULT_FPP = 0.03f) (RuntimeFilterUtil.findMinFpp), then
    BloomFilter.createEmpty(size, fpp) with BloomFilterUtil.optimalNumOfBits / optimalNumOfHashFunctions."""
    import math
    default_fpp = float(np.float32(0.03))
    n = min(max_size, max(min_size, int(ndv)))
    p = default_fpp if ndv <= 0 else max(math.exp(-3.843 * n / ndv), default_fpp)

    def java_int(x: float) -> int:  # (int) of a double: truncating, saturating
        return int(max(min(x, 2147483647.0), -2147483648.0))

    nb = java_int(-n * math.log(p) / (math.log(2) * math.log(2)))
    num_bits = nb + (64 - nb % 64)
    return num_bits, max(1, java_int(math.floor(num_bits / n * math.log(2) + 0.5)))


class BloomFilter:
    """gsql_bloom handle: the runtime filter of an INNER / SEMI hash join, bit-compatible with the reference's xxhash_64
    BloomFilter (RuntimeFilterBuilderExec puts the build keys; FilterExec's BLOOMFILTER(key) drops probe rows).  The bitmap
    is the reference's long[num_bits / 64]."""

    def __init__(self, ctx: Context, num_bits: int, num_hash_functions: int):
        self.ctx, self.num_bits, self.k = ctx, int(num_bits), int(num_hash_functions)
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_bloom_create(ctx.ptr, self.num_bits, self.k, C.byref(h)))
        self.h = h

    @property
    def nwords(self) -> int:
        return self.num_bits // 64

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_bloom_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def put(self, cols, key_col: int = 0):
        """Puts column `key_col` of every row (NULL keys put 0, as the reference's blocks do)."""
        bv = _BatchView(cols)
        self.ctx.check(self.ctx.lib.gsql_bloom_put(self.h, bv.ref(), key_col))

    def merge(self, words, nfilters: int = 1):
        """ORs `nfilters` bitmaps stored back to back (numpy uint64/int64 array, or a CUDA int64 tensor) into the filter."""
        if _is_tensor(words):
            words = words.contiguous()
            assert words.numel() == nfilters * self.nwords and words.element_size() == 8
            self.ctx.check(self.ctx.lib.gsql_bloom_merge(self.h, C.c_void_p(words.data_ptr()), nfilters, N.MEM_DEVICE))
            self.ctx.sync()
            return
        words = np.ascontiguousarray(words)
        assert words.size == nfilters * self.nwords and words.dtype.itemsize == 8
        self.ctx.check(self.ctx.lib.gsql_bloom_merge(self.h, C.c_void_p(words.ctypes.data), nfilters, N.MEM_HOST))

    def bitmap(self, mem: int = N.MEM_HOST):
        """getBitmap(): numpy uint64[num_bits / 64] (host) or a CUDA int64 tensor (device)."""
        if mem == N.MEM_DEVICE:
            out = torch.empty(self.nwords, dtype=torch.int64, device=f"cuda:{self.ctx.device}")
            self.ctx.check(self.ctx.lib.gsql_bloom_bitmap(self.h, C.c_void_p(out.data_ptr()), N.MEM_DEVICE))
            self.ctx.sync()
            return out
        out = np.empty(self.nwords, dtype=np.uint64)
        self.ctx.check(self.ctx.lib.gsql_bloom_bitmap(self.h, C.c_void_p(out.ctypes.data), N.MEM_HOST))
        return out

    def filter(self, cols, key_col: int = 0, nullable_out: Optional[bool] = None, out_cols=None):
        """BLOOMFILTER(key): -> the rows whose key might be in the filter, every column with its NULL mask, in the input's
        memory space (trimmed views of out_cols).  nullable_out=None gives an output mask exactly to the input columns
        that carry one."""
        bv = _BatchView(cols)
        cap = max(bv.rows, 1)
        wn = [nl is not None for _, nl in cols] if nullable_out is None else [nullable_out] * len(cols)
        out = out_cols if out_cols is not None else _alloc_out(self.ctx, bv.types, cap, bv.mem, wn)
        ob, _keep = _out_batch(out, bv.types, 0, bv.mem)
        n = C.c_int64()
        st = self.ctx.lib.gsql_bloom_filter(self.h, bv.ref(), key_col, C.byref(ob), cap if out_cols is None else int(out[0][0].shape[0]),
                                            C.byref(n))
        self.ctx.check(st, n.value)
        return _trim(out, n.value)


class Sort:
    """gsql_sort handle: SortExec (limit=None) or SpilledTopNExec (limit = topSize = skip + fetch) on the GPU.  Rows come out
    in the executor comparator's order: keys in turn, NULL the smallest value, DESC negating (so NULLs lead under ASC and
    trail under DESC), doubles by Double.compareTo; rows with equal keys in unspecified order."""

    def __init__(self, ctx: Context, types: Sequence[int], keys: Sequence[int], desc: Optional[Sequence[bool]] = None,
                 limit: Optional[int] = None):
        self.ctx = ctx
        self.types = list(types)
        s = N.SortSpec()
        s.n_cols = len(types)
        for i, t in enumerate(types):
            s.types[i] = t
        s.nkeys = len(keys)
        desc = list(desc) if desc is not None else [False] * len(keys)
        if len(desc) != len(keys):
            raise ValueError("one direction per key")
        for i, (k, d) in enumerate(zip(keys, desc)):
            s.key_col[i], s.key_desc[i] = k, int(bool(d))
        s.limit = -1 if limit is None else int(limit)
        self.spec = s
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_sort_create(ctx.ptr, C.byref(s), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_sort_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def consume(self, cols, rows: Optional[int] = None):
        bv = _BatchView(cols, rows)
        self.ctx.check(self.ctx.lib.gsql_sort_consume(self.h, bv.ref()))

    def finish(self) -> int:
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_sort_finish(self.h, C.byref(n)))
        return n.value

    def next(self, max_rows: int, mem: int = N.MEM_HOST, nullable_out: bool = True):
        out = _alloc_out(self.ctx, self.types, max_rows, mem, [nullable_out] * len(self.types))
        ob, _keep = _out_batch(out, self.types, 0, mem)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_sort_next(self.h, C.byref(ob), max_rows, C.byref(n)))
        if mem == N.MEM_DEVICE:
            self.ctx.sync()
        return _trim(out, n.value)

    def result(self, mem: int = N.MEM_HOST, nullable_out: bool = True):
        """finish() + every row in order."""
        n = self.finish()
        return self.next(max(n, 1), mem, nullable_out) if n > 0 else _trim(
            _alloc_out(self.ctx, self.types, 1, mem, [nullable_out] * len(self.types)), 0)


class Merge(Sort):
    """gsql_merge handle: MergeSortExec's merge of `n_inputs` runs, each already in the executor comparator's order, on
    the GPU.  consume(input, cols) appends rows to one input; the merge is stable (equal keys come out input by input,
    then in arrival order).  limit = offset + fetch: the first `limit` rows, None: every row; each input keeps at most
    `limit` rows.  finish / next / result / close as in Sort."""

    def __init__(self, ctx: Context, types: Sequence[int], key_cols: Sequence[int], desc: Optional[Sequence[bool]],
                 n_inputs: int, limit: Optional[int] = None):
        self.ctx = ctx
        self.types = list(types)
        self.n_inputs = int(n_inputs)
        s = N.SortSpec()
        s.n_cols = len(types)
        for i, t in enumerate(types):
            s.types[i] = t
        s.nkeys = len(key_cols)
        desc = list(desc) if desc is not None else [False] * len(key_cols)
        if len(desc) != len(key_cols):
            raise ValueError("one direction per key")
        for i, (k, d) in enumerate(zip(key_cols, desc)):
            s.key_col[i], s.key_desc[i] = k, int(bool(d))
        s.limit = -1 if limit is None else int(limit)
        self.spec = s
        h = C.c_void_p()
        ctx.check(ctx.lib.gsql_merge_create(ctx.ptr, C.byref(s), self.n_inputs, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.gsql_merge_destroy(self.h)
            self.h = None

    def consume(self, input: int, cols, rows: Optional[int] = None):
        bv = _BatchView(cols, rows)
        self.ctx.check(self.ctx.lib.gsql_merge_consume(self.h, int(input), bv.ref()))

    def finish(self) -> int:
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_merge_finish(self.h, C.byref(n)))
        return n.value

    def next(self, max_rows: int, mem: int = N.MEM_HOST, nullable_out: bool = True):
        out = _alloc_out(self.ctx, self.types, max_rows, mem, [nullable_out] * len(self.types))
        ob, _keep = _out_batch(out, self.types, 0, mem)
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.gsql_merge_next(self.h, C.byref(ob), max_rows, C.byref(n)))
        if mem == N.MEM_DEVICE:
            self.ctx.sync()
        return _trim(out, n.value)


def comm_unique_id() -> bytes:
    buf = (C.c_uint8 * 128)()
    st = N.load().gsql_comm_unique_id(buf)
    if st != N.OK:
        raise N.GsqlError(st, "gsql_comm_unique_id failed (NCCL not loadable?)")
    return bytes(buf)


def comm_init(ctx: Context, nranks: int, rank: int, uid: bytes):
    buf = (C.c_uint8 * 128)(*uid)
    ctx.check(ctx.lib.gsql_comm_init(ctx.ptr, nranks, rank, buf))
    ctx.nranks, ctx.rank = nranks, rank
