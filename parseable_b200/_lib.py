"""ctypes binding of include/parseable_b200.h (the C-ABI drop-in boundary).

This is the Python stand-in for the cgo/`extern "C"` binding a Parseable
maintainer would add on the Rust side (INTEGRATION.md shows that one).  It
loads the in-tree ``libparseable_b200.so`` and fails loudly when it is missing:
there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PQB_LIB: load a differently tuned build of the same library (kernel tuning experiments)
LIB_PATH = os.environ.get("PQB_LIB") or os.path.join(_HERE, "libparseable_b200.so")

PQ_OK, PQ_END_OF_STREAM = 0, 1
PQ_ERR_INVALID_ARG, PQ_ERR_UNSUPPORTED, PQ_ERR_IO, PQ_ERR_CORRUPT, PQ_ERR_CUDA, PQ_ERR_OOM = -1, -2, -3, -4, -5, -6
ERR_NAMES = {-1: "PQ_ERR_INVALID_ARG", -2: "PQ_ERR_UNSUPPORTED", -3: "PQ_ERR_IO", -4: "PQ_ERR_CORRUPT",
             -5: "PQ_ERR_CUDA", -6: "PQ_ERR_OOM"}

PQ_T_NULL, PQ_T_BOOL, PQ_T_I64, PQ_T_F64, PQ_T_UTF8, PQ_T_TS_MS = range(6)
PQ_T_DATE32 = 7   # Date32: days since 1970-01-01 in PqLiteral.i64 (6 is PQ_T_TS_NS, planning only)
PQ_OP_CMP, PQ_OP_IS_NULL, PQ_OP_IS_NOT_NULL, PQ_OP_LIKE, PQ_OP_AND, PQ_OP_OR, PQ_OP_NOT, PQ_OP_CONST, PQ_OP_REGEX, PQ_OP_IN = range(1, 11)
PQ_EQ, PQ_NE, PQ_LT, PQ_LE, PQ_GT, PQ_GE = range(6)
PQ_LIKE_NEGATED, PQ_LIKE_CASE_INSENSITIVE = 1, 2
PQ_REGEX_NEGATED, PQ_REGEX_CASE_INSENSITIVE = 1, 2
PQ_IN_NEGATED, PQ_IN_HAS_NULL = 1, 2
(PQ_AGG_COUNT_STAR, PQ_AGG_COUNT, PQ_AGG_SUM, PQ_AGG_MIN, PQ_AGG_MAX, PQ_AGG_AVG, PQ_AGG_COUNT_DISTINCT, PQ_AGG_MEDIAN,
 PQ_AGG_PERCENTILE_CONT) = range(9)
PQ_QUERY_COUNT_ONLY, PQ_QUERY_ALLREDUCE, PQ_QUERY_EMIT_ROW_IDS, PQ_QUERY_ALLGATHER = 1, 2, 4, 8
PQ_JSON_LINES = 1
PQ_COMM_ID_BYTES = 128


class PqLiteral(C.Structure):
    _fields_ = [("type", C.c_int32), ("_pad", C.c_int32), ("i64", C.c_int64), ("f64", C.c_double),
                ("str", C.c_char_p), ("str_len", C.c_uint64)]


class PqPredOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("col", C.c_int32), ("cmp", C.c_int32), ("flags", C.c_uint32),
                ("lit", PqLiteral)]


class PqAgg(C.Structure):
    _fields_ = [("fn", C.c_int32), ("col", C.c_int32)]


class PqFile(C.Structure):
    _fields_ = [("path", C.c_char_p), ("buf", C.c_void_p), ("size", C.c_uint64)]


class PqColumn(C.Structure):
    _fields_ = [("name", C.c_char_p), ("type", C.c_int32), ("_pad", C.c_int32)]


class PqKeyExpr(C.Structure):
    _fields_ = [("kind", C.c_int32), ("_pad", C.c_int32), ("width_ms", C.c_int64), ("origin_ms", C.c_int64)]


PQ_ORDER_KEY, PQ_ORDER_AGG, PQ_ORDER_COLUMN = 0, 1, 2
PQ_ORDER_DESC, PQ_ORDER_NULLS_FIRST = 1, 2


class PqOrderBy(C.Structure):
    _fields_ = [("target", C.c_int32), ("index", C.c_int32), ("flags", C.c_uint32), ("_pad", C.c_int32)]


PQ_WINDOW_ROW_NUMBER, PQ_WINDOW_PARTITION_ROWS = 1, 2


class PqWindow(C.Structure):
    _fields_ = [("partition_by", C.POINTER(PqOrderBy)), ("n_partition_by", C.c_uint32), ("flags", C.c_uint32),
                ("offset", C.c_int64), ("fetch", C.c_int64)]


class PqQueryDesc(C.Structure):
    _fields_ = [
        ("table", C.c_void_p), ("files", C.POINTER(PqFile)), ("n_files", C.c_uint32),
        ("columns", C.POINTER(PqColumn)), ("n_columns", C.c_uint32),
        ("projection", C.POINTER(C.c_int32)), ("n_projection", C.c_uint32),
        ("pred", C.POINTER(PqPredOp)), ("n_pred", C.c_uint32),
        ("group_by", C.POINTER(C.c_int32)), ("n_group_by", C.c_uint32),
        ("aggs", C.POINTER(PqAgg)), ("n_aggs", C.c_uint32),
        ("limit", C.c_int64), ("batch_size", C.c_uint32),
        ("shard_index", C.c_uint32), ("shard_count", C.c_uint32), ("flags", C.c_uint32),
        ("group_exprs", C.POINTER(PqKeyExpr)),
        ("order_by", C.POINTER(PqOrderBy)), ("n_order_by", C.c_uint32), ("_pad2", C.c_uint32),
        ("agg_params", C.POINTER(C.c_double)),
        ("window", C.POINTER(PqWindow)),
    ]


PQ_KEY_COLUMN, PQ_KEY_DATE_BIN = 0, 1

# ---- scan planning on the C side (csrc/planning.cpp) ----
PQ_T_TS_NS = 6
PQ_STAT_NONE, PQ_STAT_BOOL, PQ_STAT_INT, PQ_STAT_FLOAT, PQ_STAT_STRING = range(5)
PQ_BOUND_LOW, PQ_BOUND_HIGH, PQ_BOUND_EQ = range(3)


class PqPlanFilter(C.Structure):
    _fields_ = [("column", C.c_char_p), ("cmp", C.c_int32), ("_pad", C.c_int32), ("lit", PqLiteral)]


class PqColumnStat(C.Structure):
    _fields_ = [("column", C.c_char_p), ("kind", C.c_int32), ("_pad", C.c_int32), ("min_i", C.c_int64), ("max_i", C.c_int64),
                ("min_f", C.c_double), ("max_f", C.c_double), ("min_s", C.c_char_p), ("min_s_len", C.c_uint64),
                ("max_s", C.c_char_p), ("max_s_len", C.c_uint64)]


class PqManifestFile(C.Structure):
    _fields_ = [("path", C.c_char_p), ("num_rows", C.c_uint64), ("file_size", C.c_uint64), ("stats", C.POINTER(PqColumnStat)),
                ("n_stats", C.c_uint32), ("_pad", C.c_uint32)]


class PqManifestItem(C.Structure):
    _fields_ = [("time_lower_ns", C.c_int64), ("time_upper_ns", C.c_int64)]


class PqTimeBound(C.Structure):
    _fields_ = [("kind", C.c_int32), ("included", C.c_int32), ("time_ns", C.c_int64)]


class PqMetrics(C.Structure):
    _fields_ = [
        ("bytes_scanned", C.c_uint64), ("rows_scanned", C.c_uint64), ("rows_selected", C.c_uint64),
        ("row_groups_total", C.c_uint64), ("row_groups_pruned", C.c_uint64), ("algorithmic_bytes", C.c_uint64),
        ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("kernel_launches", C.c_uint64),
        ("device_ms", C.c_double), ("scan_kernel_ms", C.c_double), ("groups", C.c_uint64),
        ("host_ms", C.c_double), ("upload_ms", C.c_double), ("allreduce_ms", C.c_double),
        ("groups_total", C.c_uint64), ("order_ms", C.c_double), ("percentile_ms", C.c_double),
    ]

    def as_dict(self) -> dict:
        return {k: getattr(self, k) for k, _ in self._fields_}


class ArrowSchema(C.Structure):
    pass


class ArrowArray(C.Structure):
    pass


ArrowSchema._fields_ = [
    ("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
    ("n_children", C.c_int64), ("children", C.POINTER(C.POINTER(ArrowSchema))),
    ("dictionary", C.POINTER(ArrowSchema)), ("release", C.c_void_p), ("private_data", C.c_void_p)]
ArrowArray._fields_ = [
    ("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
    ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)), ("children", C.POINTER(C.POINTER(ArrowArray))),
    ("dictionary", C.POINTER(ArrowArray)), ("release", C.c_void_p), ("private_data", C.c_void_p)]

class ArrowArrayStream(C.Structure):
    _fields_ = [("get_schema", C.c_void_p), ("get_next", C.c_void_p), ("get_last_error", C.c_void_p),
                ("release", C.c_void_p), ("private_data", C.c_void_p)]


# every symbol include/parseable_b200.h declares (tests check the export list against this)
EXPORTS = [
    "pq_init", "pq_shutdown", "pq_version", "pq_device_count",
    "pq_table_open", "pq_table_rows", "pq_table_device_bytes", "pq_table_close",
    "pq_query_open", "pq_query_next", "pq_query_stream", "pq_query_json", "pq_query_metrics", "pq_last_error", "pq_query_close",
    "pq_comm_unique_id", "pq_comm_init_rank", "pq_comm_destroy",
    "pq_host_alloc", "pq_host_free", "pq_file_describe",
    "pq_plan_time_bounds", "pq_plan_manifests", "pq_plan_is_overlapping_query", "pq_plan_within_staging_window",
    "pq_plan_collect_files", "pq_plan_merge_stat", "pq_plan_pushdown",
]

_lib = None


class LibraryMissing(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load libparseable_b200.so; raises LibraryMissing (never falls back) when it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f"{LIB_PATH} is missing: run `make` (or __graft_entry__.build()). "
            "parseable_b200 has no CPU fallback for the query path.")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    lib.pq_version.restype = C.c_char_p
    lib.pq_device_count.restype = C.c_int
    lib.pq_init.argtypes = [C.POINTER(C.c_int), C.c_int]
    lib.pq_init.restype = C.c_int
    lib.pq_shutdown.restype = None
    lib.pq_table_open.argtypes = [C.POINTER(PqFile), C.c_uint32, C.POINTER(C.c_char_p), C.c_uint32,
                                  C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
    lib.pq_table_open.restype = C.c_int
    lib.pq_table_rows.argtypes = [C.c_void_p]
    lib.pq_table_rows.restype = C.c_uint64
    lib.pq_table_device_bytes.argtypes = [C.c_void_p]
    lib.pq_table_device_bytes.restype = C.c_uint64
    lib.pq_table_close.argtypes = [C.c_void_p]
    lib.pq_table_close.restype = None
    lib.pq_query_open.argtypes = [C.POINTER(PqQueryDesc), C.POINTER(C.c_void_p)]
    lib.pq_query_open.restype = C.c_int
    lib.pq_query_next.argtypes = [C.c_void_p, C.c_int, C.POINTER(ArrowArray), C.POINTER(ArrowSchema)]
    lib.pq_query_next.restype = C.c_int
    lib.pq_query_stream.argtypes = [C.c_void_p, C.c_int, C.POINTER(ArrowArrayStream)]
    lib.pq_query_stream.restype = C.c_int
    lib.pq_query_json.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    lib.pq_query_json.restype = C.c_int
    lib.pq_query_metrics.argtypes = [C.c_void_p, C.POINTER(PqMetrics)]
    lib.pq_query_metrics.restype = C.c_int
    lib.pq_last_error.argtypes = [C.c_void_p]
    lib.pq_last_error.restype = C.c_char_p
    lib.pq_query_close.argtypes = [C.c_void_p]
    lib.pq_query_close.restype = None
    lib.pq_comm_unique_id.argtypes = [C.c_char_p]
    lib.pq_comm_unique_id.restype = C.c_int
    lib.pq_comm_init_rank.argtypes = [C.c_char_p, C.c_int, C.c_int]
    lib.pq_comm_init_rank.restype = C.c_int
    lib.pq_comm_destroy.restype = C.c_int
    lib.pq_host_alloc.argtypes = [C.c_uint64]
    lib.pq_host_alloc.restype = C.c_void_p
    lib.pq_host_free.argtypes = [C.c_void_p]
    lib.pq_host_free.restype = None
    lib.pq_file_describe.argtypes = [C.POINTER(PqFile), C.c_char_p, C.c_uint64]
    lib.pq_file_describe.restype = C.c_int64
    lib.pq_plan_time_bounds.argtypes = [C.POINTER(PqPlanFilter), C.c_uint32, C.c_char_p, C.POINTER(PqTimeBound)]
    lib.pq_plan_time_bounds.restype = C.c_int32
    lib.pq_plan_manifests.argtypes = [C.POINTER(PqManifestItem), C.c_uint32, C.POINTER(PqTimeBound), C.c_uint32, C.POINTER(C.c_uint8)]
    lib.pq_plan_manifests.restype = C.c_int32
    lib.pq_plan_is_overlapping_query.argtypes = [C.POINTER(PqManifestItem), C.c_uint32, C.POINTER(PqTimeBound), C.c_uint32]
    lib.pq_plan_is_overlapping_query.restype = C.c_int32
    lib.pq_plan_within_staging_window.argtypes = [C.POINTER(PqTimeBound), C.c_uint32, C.c_int64]
    lib.pq_plan_within_staging_window.restype = C.c_int32
    lib.pq_plan_collect_files.argtypes = [C.POINTER(PqManifestFile), C.c_uint32, C.POINTER(PqPlanFilter), C.c_uint32, C.c_int64,
                                          C.POINTER(C.c_uint32)]
    lib.pq_plan_collect_files.restype = C.c_int64
    lib.pq_plan_merge_stat.argtypes = [C.POINTER(PqColumnStat), C.POINTER(PqColumnStat), C.POINTER(PqColumnStat)]
    lib.pq_plan_merge_stat.restype = C.c_int32
    lib.pq_plan_pushdown.argtypes = [C.POINTER(PqPlanFilter), C.c_uint32, C.POINTER(C.c_uint8)]
    lib.pq_plan_pushdown.restype = C.c_int32
    _lib = lib
    return lib
