"""ctypes binding of libgsql_gpu.so — the C-ABI declared in include/gsql_gpu.h.

This module is the only place that touches the shared library.  It fails loudly when the library or a CUDA
device is missing: there is no CPU fallback in this package (the CPU oracle under oracle/ is test
infrastructure and is never imported from here).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

MAX_KEYS, MAX_COLS, MAX_AGGS = 8, 32, 16
MAX_MERGE_INPUTS = 4096
T_INT32, T_INT64, T_FP64, T_DEC128 = 0, 1, 2, 3
MEM_HOST, MEM_DEVICE = 0, 1
JOIN_INNER, JOIN_LEFT, JOIN_RIGHT, JOIN_SEMI, JOIN_ANTI = 0, 1, 2, 3, 4
AGG_COUNT_STAR, AGG_COUNT, AGG_SUM, AGG_AVG, AGG_MIN, AGG_MAX, AGG_SUM0, AGG_AVG_MERGE, AGG_FIRST_VALUE = range(9)
AGG_ROW_NUMBER, AGG_RANK, AGG_DENSE_RANK = 9, 10, 11  # window functions (gsql_window only)
XCHG_HASH, XCHG_BROADCAST, XCHG_RANDOM = 0, 1, 2
OK, E_INVALID, E_CUDA, E_NCCL, E_CAPACITY, E_MORE_THAN_ONE_ROW, E_UNSUPPORTED, E_STATE, E_OOM = range(9)

TYPE_WIDTH = {T_INT32: 4, T_INT64: 8, T_FP64: 8, T_DEC128: 16}

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "_build", "libgsql_gpu.so")


class GsqlError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"gsql status {status}: {msg}")
        self.status = status


class MoreThanOneRowError(GsqlError):
    """TddlRuntimeException(ErrorCode.ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW)."""


class CapacityError(GsqlError):
    def __init__(self, status, msg, required):
        super().__init__(status, msg)
        self.required = required


class Col(C.Structure):
    _fields_ = [("type", C.c_int32), ("reserved", C.c_int32), ("data", C.c_void_p), ("nulls", C.c_void_p)]


class Batch(C.Structure):
    _fields_ = [("rows", C.c_int64), ("ncols", C.c_int32), ("mem", C.c_int32), ("cols", C.POINTER(Col))]


class JoinSpec(C.Structure):
    _fields_ = [
        ("join_type", C.c_int32), ("max_one_row", C.c_int32), ("build_outer", C.c_int32), ("nkeys", C.c_int32),
        ("outer_key", C.c_int32 * MAX_KEYS), ("inner_key", C.c_int32 * MAX_KEYS), ("key_type", C.c_int32 * MAX_KEYS),
        ("n_outer_cols", C.c_int32), ("outer_types", C.c_int32 * MAX_COLS),
        ("n_inner_cols", C.c_int32), ("inner_types", C.c_int32 * MAX_COLS),
        ("n_anti_operands", C.c_int32), ("anti_operands", C.c_int32 * MAX_KEYS),
        ("n_cond", C.c_int32), ("cond_col", C.c_int32 * 4), ("cond_ne_value", C.c_int64 * 4),
        ("expected_build_rows", C.c_int64),
    ]


class JoinInfo(C.Structure):
    _fields_ = [
        ("build_rows", C.c_int64), ("table_slots", C.c_int64), ("table_bytes", C.c_int64), ("device_bytes", C.c_int64),
        ("has_duplicate_keys", C.c_int32), ("pass_through", C.c_int32), ("pass_nothing", C.c_int32),
        ("fast_path", C.c_int32), ("partitions", C.c_int32), ("reserved", C.c_int32),
    ]


class AggCall(C.Structure):
    _fields_ = [("kind", C.c_int32), ("ncols", C.c_int32), ("cols", C.c_int32 * 4), ("filter_arg", C.c_int32)]


class DerivedCol(C.Structure):
    _fields_ = [("kind", C.c_int32), ("a", C.c_int32), ("b", C.c_int32), ("c", C.c_int32)]


MAX_DERIVED = 4
EXPR_MUL_1MINUS, EXPR_MUL_1MINUS_1PLUS = 1, 2
CMP_NONE, CMP_LE, CMP_LT, CMP_GE, CMP_GT, CMP_EQ, CMP_NE = range(7)


class AggSpec(C.Structure):
    _fields_ = [
        ("n_input_cols", C.c_int32), ("input_types", C.c_int32 * MAX_COLS),
        ("ngroups", C.c_int32), ("groups", C.c_int32 * MAX_KEYS),
        ("naggs", C.c_int32), ("aggs", AggCall * MAX_AGGS),
        ("expected_groups", C.c_int64),
        ("n_derived", C.c_int32), ("derived", DerivedCol * MAX_DERIVED),
        ("row_filter_col", C.c_int32), ("row_filter_op", C.c_int32), ("row_filter_value", C.c_int64),
    ]


MAX_SETS = 16
EXPAND_INPUT, EXPAND_NULL, EXPAND_CONST = 0, 1, 2


class ExpandItem(C.Structure):
    _fields_ = [("src", C.c_int32), ("col", C.c_int32), ("value", C.c_int64)]


class ExpandSpec(C.Structure):
    _fields_ = [
        ("n_input_cols", C.c_int32), ("input_types", C.c_int32 * MAX_COLS),
        ("nsets", C.c_int32), ("n_output_cols", C.c_int32),
        ("proj", (ExpandItem * MAX_COLS) * MAX_SETS),
    ]


class WindowSpec(C.Structure):
    _fields_ = [
        ("n_input_cols", C.c_int32), ("input_types", C.c_int32 * MAX_COLS),
        ("npart", C.c_int32), ("part_cols", C.c_int32 * MAX_KEYS),
        ("ncalls", C.c_int32), ("calls", AggCall * MAX_AGGS),
        ("reset_each_row", C.c_int32),
    ]


class XchgSpec(C.Structure):
    _fields_ = [
        ("n_cols", C.c_int32), ("types", C.c_int32 * MAX_COLS),
        ("n_channels", C.c_int32), ("channels", C.c_int32 * MAX_KEYS), ("key_types", C.c_int32 * MAX_KEYS),
        ("nparts", C.c_int32), ("mode", C.c_int32),
    ]


MAX_EXPR_INS, MAX_SCAN_OUT = 24, 16
(OP_COL, OP_CONST_I64, OP_CONST_F64, OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_NEG, OP_LT, OP_LE, OP_GT, OP_GE, OP_EQ, OP_NE,
 OP_AND, OP_OR, OP_NOT, OP_IS_NULL, OP_CAST_F64, OP_CAST_I64) = range(1, 21)
OP_CONST_NULL, OP_CASE_WHEN, OP_COALESCE, OP_BETWEEN, OP_IN = range(32, 37)  # gsql_scan_create2 only
MAX_IN_LIST, MAX_SCAN_POOL = 256, 1024


class _ExprK(C.Union):
    _fields_ = [("i", C.c_int64), ("d", C.c_double)]


class ExprIns(C.Structure):
    _fields_ = [("op", C.c_int32), ("arg", C.c_int32), ("k", _ExprK)]


class Expr(C.Structure):
    _fields_ = [("n", C.c_int32), ("reserved", C.c_int32), ("ins", ExprIns * MAX_EXPR_INS)]


class ScanSpec(C.Structure):
    _fields_ = [("n_input_cols", C.c_int32), ("input_types", C.c_int32 * MAX_COLS), ("has_filter", C.c_int32),
                ("filter", Expr), ("n_out", C.c_int32), ("reserved", C.c_int32), ("out", Expr * MAX_SCAN_OUT)]


class SortSpec(C.Structure):
    _fields_ = [("n_cols", C.c_int32), ("types", C.c_int32 * MAX_COLS), ("nkeys", C.c_int32),
                ("key_col", C.c_int32 * MAX_KEYS), ("key_desc", C.c_int32 * MAX_KEYS), ("limit", C.c_int64)]


# Every symbol include/gsql_gpu.h declares: (name, restype, argtypes).  tests/test_abi.py checks the .so exports
# each of them and that this table matches the header.
_P = C.c_void_p
_SIGS = [
    ("gsql_abi_version", C.c_int, []),
    ("gsql_ctx_create", C.c_int, [C.c_int, C.POINTER(_P)]),
    ("gsql_ctx_destroy", None, [_P]),
    ("gsql_last_error", C.c_char_p, [_P]),
    ("gsql_ctx_sync", C.c_int, [_P]),
    ("gsql_ctx_stream", _P, [_P]),
    ("gsql_ctx_set_stream", C.c_int, [_P, _P]),
    ("gsql_ctx_profile", C.c_int, [_P, C.c_int]),
    ("gsql_ctx_profile_reset", C.c_int, [_P]),
    ("gsql_ctx_profile_get", C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    ("gsql_ctx_profile_dump", C.c_int, [_P, C.c_char_p, C.c_size_t]),
    ("gsql_ctx_launch_count", C.c_int64, [_P]),
    ("gsql_host_alloc", C.c_int, [C.c_size_t, C.POINTER(_P)]),
    ("gsql_host_free", None, [_P]),
    ("gsql_device_alloc", C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    ("gsql_device_free", None, [_P, _P]),
    ("gsql_memcpy_h2d", C.c_int, [_P, _P, _P, C.c_size_t]),
    ("gsql_memcpy_d2h", C.c_int, [_P, _P, _P, C.c_size_t]),
    ("gsql_hash_rows", C.c_int, [_P, C.POINTER(Batch), C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), _P]),
    ("gsql_partition_ids", C.c_int, [_P, _P, C.c_int64, C.c_int32, _P, C.c_int32]),
    ("gsql_join_create", C.c_int, [_P, C.POINTER(JoinSpec), C.POINTER(_P)]),
    ("gsql_join_build_consume", C.c_int, [_P, C.POINTER(Batch)]),
    ("gsql_join_build_consume_ref", C.c_int, [_P, C.POINTER(Batch)]),
    ("gsql_join_build_finish", C.c_int, [_P]),
    ("gsql_join_info_get", C.c_int, [_P, C.POINTER(JoinInfo)]),
    ("gsql_join_output_schema", C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("gsql_join_probe_count", C.c_int, [_P, C.POINTER(Batch), C.POINTER(C.c_int64)]),
    ("gsql_join_probe", C.c_int, [_P, C.POINTER(Batch), C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_join_unmatched_build", C.c_int, [_P, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_join_destroy", None, [_P]),
    ("gsql_agg_create", C.c_int, [_P, C.POINTER(AggSpec), C.POINTER(_P)]),
    ("gsql_agg_consume", C.c_int, [_P, C.POINTER(Batch)]),
    ("gsql_agg_finish", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("gsql_agg_output_schema", C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("gsql_agg_next", C.c_int, [_P, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_agg_destroy", None, [_P]),
    ("gsql_gsagg_create", C.c_int, [_P, C.POINTER(ExpandSpec), C.POINTER(AggSpec), C.POINTER(_P)]),
    ("gsql_gsagg_consume", C.c_int, [_P, C.POINTER(Batch)]),
    ("gsql_gsagg_finish", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("gsql_gsagg_output_schema", C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("gsql_gsagg_next", C.c_int, [_P, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_gsagg_destroy", None, [_P]),
    ("gsql_sortagg_create", C.c_int, [_P, C.POINTER(AggSpec), C.POINTER(_P)]),
    ("gsql_sortagg_consume", C.c_int, [_P, C.POINTER(Batch), C.POINTER(C.c_int64)]),
    ("gsql_sortagg_finish", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("gsql_sortagg_output_schema", C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("gsql_sortagg_next", C.c_int, [_P, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_sortagg_destroy", None, [_P]),
    ("gsql_window_create", C.c_int, [_P, C.POINTER(WindowSpec), C.POINTER(_P)]),
    ("gsql_window_output_schema", C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("gsql_window_apply", C.c_int, [_P, C.POINTER(Batch), C.POINTER(Batch)]),
    ("gsql_window_destroy", None, [_P]),
    ("gsql_scan_create", C.c_int, [_P, C.POINTER(ScanSpec), C.POINTER(_P)]),
    ("gsql_scan_create2", C.c_int, [_P, C.POINTER(ScanSpec), C.POINTER(C.c_int64), C.c_int32, C.POINTER(_P)]),
    ("gsql_scan_output_schema", C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("gsql_scan_apply", C.c_int, [_P, C.POINTER(Batch), C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_scan_destroy", None, [_P]),
    ("gsql_xchg_create", C.c_int, [_P, C.POINTER(XchgSpec), C.POINTER(_P)]),
    ("gsql_xchg_partition", C.c_int, [_P, C.POINTER(Batch), C.POINTER(Batch), C.POINTER(C.c_int64)]),
    ("gsql_comm_unique_id", C.c_int, [C.POINTER(C.c_uint8)]),
    ("gsql_comm_init", C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_uint8)]),
    ("gsql_comm_destroy", C.c_int, [_P]),
    ("gsql_xchg_open_p2p", C.c_int, [_P, C.c_int64, C.c_uint32]),
    ("gsql_xchg_push", C.c_int, [_P, C.POINTER(Batch), C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("gsql_xchg_recv_view", C.c_int, [_P, C.c_int32, C.POINTER(Batch)]),
    ("gsql_xchg_push_wait", C.c_int, [_P]),
    ("gsql_xchg_plan_layout", C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                          C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("gsql_xchg_destroy", None, [_P]),
    ("gsql_serde_size", C.c_int, [_P, C.POINTER(Batch), C.c_int32, C.POINTER(C.c_int64)]),
    ("gsql_serde_serialize", C.c_int, [_P, C.POINTER(Batch), C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_serde_deserialize", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_bloom_create", C.c_int, [_P, C.c_int64, C.c_int32, C.POINTER(_P)]),
    ("gsql_bloom_put", C.c_int, [_P, C.POINTER(Batch), C.c_int32]),
    ("gsql_bloom_merge", C.c_int, [_P, _P, C.c_int64, C.c_int32]),
    ("gsql_bloom_bitmap", C.c_int, [_P, _P, C.c_int32]),
    ("gsql_bloom_filter", C.c_int, [_P, C.POINTER(Batch), C.c_int32, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_bloom_destroy", None, [_P]),
    ("gsql_sort_create", C.c_int, [_P, C.POINTER(SortSpec), C.POINTER(_P)]),
    ("gsql_sort_consume", C.c_int, [_P, C.POINTER(Batch)]),
    ("gsql_sort_finish", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("gsql_sort_next", C.c_int, [_P, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_sort_destroy", None, [_P]),
    ("gsql_merge_create", C.c_int, [_P, C.POINTER(SortSpec), C.c_int32, C.POINTER(_P)]),
    ("gsql_merge_consume", C.c_int, [_P, C.c_int32, C.POINTER(Batch)]),
    ("gsql_merge_finish", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("gsql_merge_next", C.c_int, [_P, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_merge_destroy", None, [_P]),
    ("gsql_smj_create", C.c_int, [_P, C.POINTER(JoinSpec), C.POINTER(C.c_int32), C.POINTER(_P)]),
    ("gsql_smj_inner_consume", C.c_int, [_P, C.POINTER(Batch)]),
    ("gsql_smj_inner_finish", C.c_int, [_P]),
    ("gsql_smj_output_schema", C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("gsql_smj_probe", C.c_int, [_P, C.POINTER(Batch), C.POINTER(C.c_int64)]),
    ("gsql_smj_next", C.c_int, [_P, C.POINTER(Batch), C.c_int64, C.POINTER(C.c_int64)]),
    ("gsql_smj_destroy", None, [_P]),
]
ABI_SYMBOLS = [s[0] for s in _SIGS]

_lib: Optional[C.CDLL] = None


def load(path: Optional[str] = None) -> C.CDLL:
    """dlopen libgsql_gpu.so and bind every ABI symbol.  Raises if the extension was not built."""
    global _lib
    if _lib is not None:
        return _lib
    path = path or SO_PATH
    if not os.path.exists(path):
        raise ImportError(
            f"{path} is missing: build it with `python -m galaxysql_b200.build` (or __graft_entry__.build()). "
            "galaxysql_b200 has no CPU fallback.")
    lib = C.CDLL(path)
    for name, res, args in _SIGS:
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(ctx_ptr, status: int, required: Optional[int] = None):
    if status == OK:
        return
    msg = load().gsql_last_error(ctx_ptr).decode(errors="replace") if ctx_ptr else ""
    if status == E_MORE_THAN_ONE_ROW:
        raise MoreThanOneRowError(status, msg)
    if status == E_CAPACITY:
        raise CapacityError(status, msg, required)
    raise GsqlError(status, msg)
