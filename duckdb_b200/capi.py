"""ctypes binding of the C ABI in include/duckdb_b200.h (libduckdb_b200.so).

This is the only way Python code (tests, bench, the host-side operator mirror in
operators.py) reaches the CUDA kernels: plain pointers and sizes, exactly what
the DuckDB-side C++ shim (integration/) passes.  There is no CPU fallback: if the
library is missing or no CUDA device is usable, calls raise B200Error.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libduckdb_b200.so")

OK = 0
ERR_INVALID, ERR_NO_DEVICE, ERR_CUDA, ERR_OOM, ERR_OVERFLOW, ERR_CAPACITY = -1, -2, -3, -4, -5, -6

# b200_type
BOOL, UINT8, INT8, UINT16, INT16, UINT32, INT32, UINT64, INT64 = 1, 2, 3, 4, 5, 6, 7, 8, 9
FLOAT, DOUBLE, INT128 = 11, 12, 204
FLAT_VECTOR, CONSTANT_VECTOR, DICTIONARY_VECTOR = 0, 2, 3

TYPE_OF_DTYPE = {
    np.dtype(np.bool_): BOOL, np.dtype(np.uint8): UINT8, np.dtype(np.int8): INT8,
    np.dtype(np.uint16): UINT16, np.dtype(np.int16): INT16, np.dtype(np.uint32): UINT32,
    np.dtype(np.int32): INT32, np.dtype(np.uint64): UINT64, np.dtype(np.int64): INT64,
    np.dtype(np.float32): FLOAT, np.dtype(np.float64): DOUBLE,
}
DTYPE_OF_TYPE = {v: k for k, v in TYPE_OF_DTYPE.items()}
TYPE_SIZE = {BOOL: 1, UINT8: 1, INT8: 1, UINT16: 2, INT16: 2, UINT32: 4, INT32: 4, UINT64: 8, INT64: 8,
             FLOAT: 4, DOUBLE: 8, INT128: 16}

# expression opcodes (b200_expr_op)
EXPR_COLREF, EXPR_CONST = 227, 75
EXPR_NOT, EXPR_IS_NULL, EXPR_IS_NOT_NULL = 13, 14, 15
EXPR_EQ, EXPR_NE, EXPR_LT, EXPR_GT, EXPR_LE, EXPR_GE = 25, 26, 27, 28, 29, 30
EXPR_DISTINCT, EXPR_NOT_DISTINCT = 37, 40
EXPR_AND, EXPR_OR = 50, 51
EXPR_ADD, EXPR_SUB, EXPR_MUL, EXPR_CAST = 1001, 1002, 1003, 1004

AGG_COUNT_STAR, AGG_COUNT, AGG_SUM, AGG_SUM_NO_OVERFLOW, AGG_MIN, AGG_MAX, AGG_AVG = 0, 1, 2, 3, 4, 5, 6
JOIN_LEFT, JOIN_INNER, JOIN_SEMI, JOIN_ANTI, JOIN_MARK = 1, 3, 5, 6, 7
JOIN_RIGHT, JOIN_OUTER = 2, 4


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[b200 status {code}] {msg}")
        self.code = code


class Vector(C.Structure):
    _fields_ = [("type", C.c_int32), ("vector_type", C.c_int32), ("data", C.c_void_p),
                ("sel", C.c_void_p), ("validity", C.c_void_p), ("dict_size", C.c_uint64)]


class _Val(C.Union):
    _fields_ = [("i", C.c_int64), ("u", C.c_uint64), ("d", C.c_double), ("f", C.c_float)]


class ExprNode(C.Structure):
    _fields_ = [("op", C.c_int32), ("type", C.c_int32), ("left", C.c_int32), ("right", C.c_int32),
                ("col", C.c_int32), ("is_null", C.c_int32), ("value", _Val)]


class AggDesc(C.Structure):
    _fields_ = [("func", C.c_int32), ("input_type", C.c_int32), ("input", C.c_int32), ("reserved", C.c_int32)]


_lib = None


def lib():
    """Load libduckdb_b200.so (fails loudly when it was not built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200Error(ERR_INVALID, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`"
                                     " (there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, u64p, i32p = C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)
    intp = C.POINTER(C.c_int)
    L.b200_last_error.restype = C.c_char_p
    L.b200_version.restype = C.c_char_p
    L.b200_device_count.restype = C.c_int
    L.b200_ctx_create.argtypes = [C.c_int, vp, C.POINTER(vp)]
    L.b200_ctx_destroy.argtypes = [vp]
    L.b200_ctx_destroy.restype = None
    L.b200_ctx_sync.argtypes = [vp]
    L.b200_ctx_stats.argtypes = [vp, u64p, u64p, u64p]
    L.b200_host_alloc.argtypes = [vp, C.c_size_t, C.POINTER(vp)]
    L.b200_host_free.argtypes = [vp, vp]
    L.b200_host_trim.argtypes = []
    L.b200_batch_upload.argtypes = [vp, C.POINTER(Vector), C.c_int, C.c_uint64, C.POINTER(vp)]
    L.b200_batch_upload_to.argtypes = [vp, C.POINTER(Vector), C.c_int, C.c_uint64, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.b200_batch_wrap.argtypes = [vp, C.POINTER(Vector), C.c_int, C.c_uint64, C.POINTER(vp)]
    L.b200_batch_rows.argtypes = [vp]
    L.b200_batch_rows.restype = C.c_uint64
    L.b200_batch_cols.argtypes = [vp]
    L.b200_batch_column.argtypes = [vp, C.c_int, C.POINTER(Vector)]
    L.b200_batch_download.argtypes = [vp, vp, C.c_int, vp, vp]
    L.b200_batch_free.argtypes = [vp]
    L.b200_batch_free.restype = None
    L.b200_hash.argtypes = [vp, vp, intp, C.c_int, vp]
    L.b200_filter_project.argtypes = [vp, vp, C.POINTER(ExprNode), C.c_int, C.c_int, intp, C.c_int, C.POINTER(vp),
                                      vp, vp, u64p]
    L.b200_agg_create.argtypes = [vp, i32p, C.c_int, C.POINTER(AggDesc), C.c_int, C.c_uint64, C.POINTER(vp)]
    L.b200_agg_create_filtered.argtypes = [vp, i32p, C.c_int, C.POINTER(AggDesc), i32p, C.c_int, C.c_uint64,
                                           C.POINTER(vp)]
    L.b200_agg_sink.argtypes = [vp, vp, intp, intp]
    L.b200_agg_group_count.argtypes = [vp, u64p]
    L.b200_agg_export_states.argtypes = [vp, C.POINTER(vp)]
    L.b200_agg_combine_states.argtypes = [vp, vp]
    L.b200_agg_packed_words.argtypes = [vp, C.c_uint64]
    L.b200_agg_packed_words.restype = C.c_uint64
    L.b200_agg_export_packed.argtypes = [vp, vp, C.c_uint64]
    L.b200_agg_combine_packed.argtypes = [vp, vp, C.c_int, C.c_uint64]
    L.b200_agg_finalize.argtypes = [vp, C.POINTER(vp)]
    L.b200_agg_destroy.argtypes = [vp]
    L.b200_agg_destroy.restype = None
    L.b200_join_create.argtypes = [vp, C.c_int, i32p, C.c_int, i32p, C.c_int, C.POINTER(vp)]
    L.b200_join_build_sink.argtypes = [vp, vp, intp, intp]
    L.b200_join_finalize.argtypes = [vp]
    L.b200_join_build_rows.argtypes = [vp, u64p]
    L.b200_join_probe.argtypes = [vp, vp, intp, intp, C.c_int, C.c_uint64, C.POINTER(vp), vp, u64p]
    L.b200_join_probe_mark.argtypes = [vp, vp, intp, vp, vp]
    L.b200_join_scan_unmatched.argtypes = [vp, C.c_uint64, C.c_uint64, C.POINTER(vp), vp, u64p]
    L.b200_join_destroy.argtypes = [vp]
    L.b200_join_destroy.restype = None
    L.b200_radix_partition.argtypes = [vp, vp, intp, C.c_int, C.c_int, C.POINTER(vp), u64p]
    L.b200_partition_count.argtypes = [vp, vp, intp, C.c_int, C.c_int, u64p]
    L.b200_partition_scatter.argtypes = [vp, vp, intp, C.c_int, C.c_int, C.POINTER(vp), u64p]
    L.b200_partition_count_dev.argtypes = [vp, vp, intp, C.c_int, C.c_int, vp]
    L.b200_partition_scatter_dev.argtypes = [vp, vp, intp, C.c_int, C.c_int, C.POINTER(vp), vp, C.c_uint64, vp]
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "b200_last_error", "b200_version", "b200_device_count", "b200_ctx_create", "b200_ctx_destroy", "b200_ctx_sync",
    "b200_ctx_stats", "b200_host_alloc", "b200_host_free", "b200_host_trim", "b200_batch_upload", "b200_batch_upload_to", "b200_batch_wrap", "b200_batch_rows",
    "b200_batch_cols", "b200_batch_column", "b200_batch_download", "b200_batch_free", "b200_hash",
    "b200_filter_project", "b200_agg_create", "b200_agg_create_filtered", "b200_agg_sink", "b200_agg_group_count", "b200_agg_export_states",
    "b200_agg_combine_states", "b200_agg_packed_words", "b200_agg_export_packed", "b200_agg_combine_packed",
    "b200_agg_finalize", "b200_agg_destroy", "b200_join_create", "b200_join_build_sink",
    "b200_join_finalize", "b200_join_build_rows", "b200_join_probe", "b200_join_probe_mark", "b200_join_scan_unmatched", "b200_join_destroy", "b200_radix_partition",
    "b200_partition_count", "b200_partition_scatter", "b200_partition_count_dev", "b200_partition_scatter_dev",
]


def check(rc):
    if rc != OK:
        msg = lib().b200_last_error()
        raise B200Error(rc, msg.decode() if msg else "")


def int_array(values):
    return (C.c_int * max(1, len(values)))(*values)


def i32_array(values):
    return (C.c_int32 * max(1, len(values)))(*values)


def validity_words(valid):
    """bool array -> DuckDB ValidityMask words (uint64, bit=1 valid)."""
    n = len(valid)
    bits = np.zeros(((n + 63) // 64) * 64, dtype=np.uint8)
    bits[:n] = valid
    return np.packbits(bits, bitorder="little").view(np.uint64).copy()


def valid_from_words(words, n):
    return np.unpackbits(np.ascontiguousarray(words).view(np.uint8), bitorder="little")[:n].astype(bool)
