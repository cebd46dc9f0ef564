"""ctypes binding of include/spark_b200.h -- the same symbols the JNI shim binds (INTEGRATION.md).

There is no CPU fallback: if libsparkb200.so is missing, fails to load, or no H100 is visible,
every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsparkb200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "spark_b200.h")

# ---- constants (mirrors of the #defines) -------------------------------------------------------
SB_OK = 0
(SB_BOOL, SB_INT8, SB_INT16, SB_INT32, SB_INT64, SB_FLOAT32, SB_FLOAT64, SB_DATE32, SB_TIMESTAMP, SB_DECIMAL64,
 SB_STRING, SB_DECIMAL128) = range(1, 13)
SB_OP = dict(COL=1, LIT_I64=2, LIT_F64=3, LIT_NULL=4, ADD=10, SUB=11, MUL=12, DIV=13, NEG=14, EQ=20, NE=21, LT=22,
             LE=23, GT=24, GE=25, AND=30, OR=31, NOT=32, ISNULL=33, ISNOTNULL=34, CAST_F64=40, CAST_I64=41, CAST_I32=42,
             STR_EQ=50, STR_LT=51, STR_LE=52, STR_GT=53, STR_GE=54, STR_IN=55, STR_STARTS_WITH=56, STR_ENDS_WITH=57, STR_CONTAINS=58,
             STR_LIKE=59, STR_OCTET_LENGTH=60, STR_CHAR_LENGTH=61,
             SF_COL=70, SF_LIT=71, SF_SUBSTRING=72, SF_CONCAT=73, SF_CONCAT_WS=74, SF_TRIM=75, SF_LTRIM=76, SF_RTRIM=77, SF_LPAD=78,
             SF_RPAD=79)
SB_SF_MAX_RANGES = 16
SB_VT_BOOL, SB_VT_I32, SB_VT_I64, SB_VT_F64 = 1, 2, 3, 4
SB_AGG = dict(sum=1, avg=2, count=3, count_star=4, min=5, max=6, var_pop=7, var_samp=8, stddev_pop=9, stddev_samp=10)
SB_AGG_FLAG_NAN_ON_DIVIDE_BY_ZERO = 1
SB_AGG_MODE = dict(partial=1, final=2, complete=3, partial_merge=4)
SB_JOIN = dict(inner=0, left_outer=1, left_semi=2, left_anti=3, full_outer=4, build_outer=5, existence=6, left_anti_null_aware=7)
SB_UNIQUE_ID_BYTES = 128

def decimal_type(precision, scale):
    """sb_column.scale word of a decimal column: SB_DECIMAL_TYPE(precision, scale)"""
    return (precision << 8) | scale


TYPE_WIDTH = {SB_BOOL: 1, SB_INT8: 1, SB_INT16: 2, SB_INT32: 4, SB_INT64: 8, SB_FLOAT32: 4, SB_FLOAT64: 8,
              SB_DATE32: 4, SB_TIMESTAMP: 8, SB_DECIMAL64: 8, SB_STRING: 0, SB_DECIMAL128: 16}


class sb_column(C.Structure):
    _fields_ = [("type", C.c_int32), ("scale", C.c_int32), ("length", C.c_int64), ("null_count", C.c_int64),
                ("data", C.c_void_p), ("validity", C.c_void_p), ("offsets", C.c_void_p)]


class sb_page(C.Structure):
    _fields_ = [("encoding", C.c_int32), ("num_values", C.c_int32), ("values_offset", C.c_int64), ("values_bytes", C.c_int64),
                ("def_offset", C.c_int64), ("def_bytes", C.c_int64)]


class sb_column_chunk(C.Structure):
    _fields_ = [("type", C.c_int32), ("scale", C.c_int32), ("physical_type", C.c_int32), ("npages", C.c_int32), ("data", C.c_void_p),
                ("data_bytes", C.c_int64), ("pages", C.POINTER(sb_page)), ("dict_offset", C.c_int64), ("dict_count", C.c_int32), ("value_multiplier", C.c_int32)]


class sb_page_span(C.Structure):
    _fields_ = [("page_type", C.c_int32), ("encoding", C.c_int32), ("num_values", C.c_int32), ("levels_bytes", C.c_int32),
                ("body_offset", C.c_int64), ("compressed_bytes", C.c_int32), ("uncompressed_bytes", C.c_int32),
                ("values_compressed", C.c_int32), ("header_bytes", C.c_int32)]


class sb_compressed_chunk(C.Structure):
    _fields_ = [("type", C.c_int32), ("scale", C.c_int32), ("physical_type", C.c_int32), ("codec", C.c_int32),
                ("max_def_level", C.c_int32), ("npages", C.c_int32), ("value_multiplier", C.c_int32), ("pad", C.c_int32),
                ("data", C.c_void_p), ("data_bytes", C.c_int64),
                ("spans", C.POINTER(sb_page_span))]


# parquet.thrift CompressionCodec; the GPU scan decodes UNCOMPRESSED and SNAPPY
SB_CODEC = dict(UNCOMPRESSED=0, SNAPPY=1, GZIP=2, LZO=3, BROTLI=4, LZ4=5, ZSTD=6, LZ4_RAW=7)

SB_ENC_PLAIN, SB_ENC_RLE_DICTIONARY, SB_ENC_RLE_BOOLEAN = 0, 1, 2
SB_ENC_DELTA_BINARY_PACKED, SB_ENC_DELTA_LENGTH_BYTE_ARRAY, SB_ENC_DELTA_BYTE_ARRAY = 3, 4, 5
SB_PHYS = dict(BOOLEAN=0, INT32=1, INT64=2, FLOAT=4, DOUBLE=5, BYTE_ARRAY=6)


class _lit(C.Union):
    _fields_ = [("i", C.c_int64), ("d", C.c_double)]


class sb_expr_node(C.Structure):
    _fields_ = [("op", C.c_int32), ("vtype", C.c_int32), ("arg", C.c_int32), ("arg2", C.c_int32), ("lit", _lit)]


class sb_expr(C.Structure):
    _fields_ = [("nodes", C.POINTER(sb_expr_node)), ("n", C.c_int32), ("out_type", C.c_int32), ("bytes", C.c_void_p), ("nbytes", C.c_int64)]


class sb_agg_spec(C.Structure):
    _fields_ = [("func", C.c_int32), ("flags", C.c_int32), ("input", sb_expr)]


class sb_agg_plan(C.Structure):
    _fields_ = [("mode", C.c_int32), ("nkeys", C.c_int32), ("key_cols", C.POINTER(C.c_int32)), ("naggs", C.c_int32),
                ("pad", C.c_int32), ("aggs", C.POINTER(sb_agg_spec)), ("filter", C.POINTER(sb_expr)),
                ("expected_groups", C.c_int64)]


class sb_join_options(C.Structure):
    _fields_ = [("probe_filter", C.POINTER(sb_expr)), ("condition", C.POINTER(sb_expr)), ("probe_out_cols", C.POINTER(C.c_int32)),
                ("n_probe_out", C.c_int32), ("n_build_out", C.c_int32), ("build_out_cols", C.POINTER(C.c_int32)),
                ("n_runtime_filters", C.c_int32), ("runtime_filter_cols", C.POINTER(C.c_int32)), ("runtime_filter_relations", C.POINTER(C.c_void_p))]


class sb_sort_order(C.Structure):
    _fields_ = [("col", C.c_int32), ("ascending", C.c_int32), ("nulls_first", C.c_int32), ("pad", C.c_int32)]


class sb_window_spec(C.Structure):
    _fields_ = [("func", C.c_int32), ("col", C.c_int32), ("frame_type", C.c_int32), ("pad", C.c_int32), ("lower", C.c_int64),
                ("upper", C.c_int64), ("param", C.c_int64)]


SB_WIN = {"row_number": 1, "rank": 2, "dense_rank": 3, "percent_rank": 4, "cume_dist": 5, "ntile": 6, "lag": 7, "lead": 8, "sum": 9,
          "count": 10, "avg": 11, "min": 12, "max": 13, "first_value": 14, "last_value": 15}
SB_FRAME_ROWS, SB_FRAME_RANGE, SB_FRAME_RANGE_F64 = 0, 1, 2
SB_UNBOUNDED_PRECEDING, SB_UNBOUNDED_FOLLOWING = -(1 << 63), (1 << 63) - 1


class SparkB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libsparkb200 error %d: %s" % (code, msg))
        self.code = code


_lib = None
_initialized_device = None

_p = C.c_void_p
_pp = C.POINTER(C.c_void_p)
_i32, _i64 = C.c_int32, C.c_int64

# symbol -> argtypes (return type is int unless listed in _RESTYPE)
_SIGNATURES = {
    "sb_init": [_i32], "sb_shutdown": [], "sb_last_error": [], "sb_abi_version": [],
    "sb_device_info": [C.POINTER(_i64)], "sb_kernel_launch_count": [],
    "sb_config_set": [C.c_char_p, _i64], "sb_config_get": [C.c_char_p, C.POINTER(_i64)], "sb_hash_aggregate_last_plan": [],
    "sb_agg_rtc_compile_check": [C.POINTER(_i32), _i32, C.c_char_p, _i32], "sb_agg_plan_meta_words": [],
    "sb_profile_dump": [C.c_char_p, _i32],
    "sb_profile_enable": [_i32], "sb_profile_reset": [], "sb_profile_get": [C.c_char_p, C.POINTER(C.c_double), C.POINTER(_i64)],
    "sb_host_alloc": [_i64, _pp], "sb_host_free": [_p],
    "sb_stream_create": [_pp], "sb_stream_destroy": [_p], "sb_stream_synchronize": [_p],
    "sb_stream_record_start": [_p], "sb_stream_record_stop": [_p], "sb_stream_elapsed_ms": [_p, C.POINTER(C.c_float)],
    "sb_table_import_host": [C.POINTER(sb_column), _i32, _p, _pp],
    "sb_table_import_device": [C.POINTER(sb_column), _i32, _pp],
    "sb_table_num_rows": [_p, C.POINTER(_i64)], "sb_table_num_columns": [_p, C.POINTER(_i32)],
    "sb_table_column": [_p, _i32, C.POINTER(sb_column)], "sb_table_string_bytes": [_p, _i32, C.POINTER(_i64)],
    "sb_table_export_host": [_p, _i32, _p, _p, _p, C.POINTER(_i64), _p],
    "sb_table_retain": [_p], "sb_table_release": [_p],
    "sb_table_select": [_p, C.POINTER(_i32), _i32, _pp], "sb_table_zip": [_p, _p, _pp],
    "sb_table_slice": [_p, _i64, _i64, _p, _pp], "sb_table_concat": [_pp, _i32, _p, _pp],
    "sb_dictionary_encode": [_p, _i32, _p, _pp, _pp], "sb_dictionary_lookup": [_p, _i32, _p, _p, _pp],
    "sb_dictionary_decode": [_p, _i32, _p, _p, _pp],
    "sb_window": [_p, C.POINTER(C.c_int32), _i32, C.POINTER(sb_sort_order), _i32, C.POINTER(sb_window_spec), _i32, _p, _pp], "sb_expand": [_p, _p, _i32, _i32, _p, _pp],
    "sb_parquet_chunk_pages": [_p, _i64, _i32, C.POINTER(sb_page), _i32, C.POINTER(_i32), C.POINTER(_i64), C.POINTER(_i32)],
    "sb_scan_decode": [C.POINTER(sb_column_chunk), _i32, _p, _pp],
    "sb_parquet_page_spans": [_p, _i64, _i32, _i32, C.POINTER(sb_page_span), _i32, C.POINTER(_i32)],
    "sb_scan_decode_compressed": [C.POINTER(sb_compressed_chunk), _i32, _p, _pp],
    "sb_scan_encode": [_p, _i32, _p, _i64, _p, _pp, C.POINTER(sb_page), _i32, C.POINTER(_i32), C.POINTER(_i64), C.POINTER(_i32)],
    "sb_filter_project": [_p, C.POINTER(sb_expr), C.POINTER(sb_expr), _i32, _p, _pp],
    "sb_string_project": [_p, C.POINTER(sb_expr), _i32, _p, _pp],
    "sb_partition_ids": [_p, C.POINTER(_i32), _i32, _i32, _p, _p],
    "sb_hash_partition": [_p, C.POINTER(_i32), _i32, _i32, _p, _pp, C.POINTER(_i64)],
    "sb_round_robin_partition": [_p, _i32, _i32, _p, _pp, C.POINTER(_i64)],
    "sb_range_partition": [_p, C.POINTER(sb_sort_order), _p, _p, _pp, C.POINTER(_i64)],
    "sb_range_sample": [_p, C.POINTER(sb_sort_order), _i64, C.c_uint64, _p, _pp],
    "sb_range_determine_bounds": [_p, C.POINTER(sb_sort_order), _i32, _p, _pp],
    "sb_hash_aggregate": [_p, C.POINTER(sb_agg_plan), _p, _pp],
    "sb_hash_agg_create": [C.POINTER(sb_agg_plan), _pp], "sb_hash_agg_update": [_p, _p, _p],
    "sb_hash_agg_merge": [_p, _p, _p], "sb_hash_agg_finish": [_p, _p, _pp], "sb_hash_agg_destroy": [_p],
    "sb_synth_table": [_i32, C.POINTER(_i32), _i32, _i64, _i64, _i64, C.c_uint64, _p, _pp],
    "sb_sort": [_p, C.POINTER(sb_sort_order), _i32, _p, _pp],
    "sb_sort_permutation": [_p, C.POINTER(sb_sort_order), _i32, _p, _p],
    "sb_top_n": [_p, C.POINTER(sb_sort_order), _i32, _i64, _p, _pp],
    "sb_join_build": [_p, C.POINTER(_i32), _i32, _p, _pp],
    "sb_join_probe": [_p, _p, C.POINTER(_i32), _i32, _i32, _p, _pp],
    "sb_join_build_filtered": [_p, C.POINTER(_i32), _i32, C.POINTER(sb_expr), _p, _pp],
    "sb_join_probe_ex": [_p, _p, C.POINTER(_i32), _i32, _i32, C.POINTER(sb_join_options), _p, _pp],
    "sb_join_probe_condition": [_p, _p, C.POINTER(_i32), _i32, _i32, C.POINTER(sb_expr), _p, _pp],
    "sb_hash_table_release": [_p],
    "sb_comm_get_unique_id": [C.c_char_p], "sb_comm_init": [_i32, _i32, C.c_char_p], "sb_comm_destroy": [],
    "sb_comm_rank": [C.POINTER(_i32), C.POINTER(_i32)],
    "sb_exchange_plan": [C.POINTER(_i64), _i32, _i32, C.POINTER(_i64)],
    "sb_all_to_all": [_p, C.POINTER(_i64), _i32, _p, _pp, C.POINTER(_i64)],
    "sb_all_gather": [_p, _p, _pp],
    "sb_shuffle_exchange": [_p, C.POINTER(_i32), _i32, _i32, _p, _pp, C.POINTER(_i64)],
    "sb_exchange_counts": [C.POINTER(_i64), _i32, _p, C.POINTER(_i64)],
    "sb_map_output_statistics": [_p, C.POINTER(_i64), _i32, _p, C.POINTER(_i64)],
    "sb_coalesce_partitions": [C.POINTER(C.POINTER(_i64)), _i32, _i32, _i64, _i32, _i64, _i32, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i64),
                               C.POINTER(_i32)],
}
_RESTYPE = {"sb_agg_plan_meta_words": _i32, "sb_hash_aggregate_last_plan": C.c_char_p, "sb_last_error": C.c_char_p, "sb_abi_version": _i32, "sb_kernel_launch_count": _i64}


def declared_symbols():
    """Every function name include/spark_b200.h declares (used by the CPU test that the .so exports them)."""
    with open(HEADER_PATH) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sb_[a-z0-9_]+)\s*\(", text)))


def _preload_nccl():
    """libsparkb200 resolves NCCL with dlopen("libnccl.so.2") when a communicator is first needed.  In a Python process that
    also imports torch LATER, the loader would hand torch whatever libnccl.so.2 is already mapped -- the system copy (2.27) instead
    of the newer one torch bundles and needs (undefined symbol ncclDevCommCreate).  Mapping torch's bundled copy first makes both
    sides share it.  A JVM executor has no such neighbour and simply uses the system library."""
    try:
        import importlib.util
        spec = importlib.util.find_spec("nvidia")
        for base in (list(spec.submodule_search_locations) if spec and spec.submodule_search_locations else []):
            cand = os.path.join(base, "nccl", "lib", "libnccl.so.2")
            if os.path.exists(cand):
                C.CDLL(cand, mode=C.RTLD_GLOBAL)
                return cand
    except Exception:
        pass
    return None


def load():
    """dlopen libsparkb200.so and attach signatures.  Raises if the extension has not been built."""
    global _lib
    if _lib is None:
        _preload_nccl()
        if not os.path.exists(LIB_PATH):
            raise SparkB200Error(-1, "libsparkb200.so is not built (run `python -m spark_b200.build`); there is no CPU fallback")
        lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, args in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = _RESTYPE.get(name, C.c_int)
        _lib = lib
    return _lib


def check(code):
    if code != SB_OK:
        raise SparkB200Error(code, load().sb_last_error().decode("utf-8", "replace"))


def init(device_ordinal=None):
    """sb_init on the device of this process (LOCAL_RANK under torchrun).  Idempotent."""
    global _initialized_device
    lib = load()
    if device_ordinal is None:
        device_ordinal = int(os.environ.get("LOCAL_RANK", "0"))
    if _initialized_device is None:
        check(lib.sb_init(device_ordinal))
        _initialized_device = device_ordinal
    return lib


def kernel_launch_count():
    return int(load().sb_kernel_launch_count())


def config_set(key: str, value: int):
    check(load().sb_config_set(key.encode(), int(value)))


def config_get(key: str) -> int:
    v = _i64()
    check(load().sb_config_get(key.encode(), C.byref(v)))
    return int(v.value)


def profile_dump() -> dict:
    """{section: (total_ms, launches)} of every device-timed section since sb_profile_reset."""
    buf = C.create_string_buffer(1 << 14)
    check(load().sb_profile_dump(buf, len(buf)))
    out = {}
    for item in buf.value.decode().split(";"):
        if "=" in item:
            k, v = item.split("=")
            ms, n = v.split("/")
            out[k] = (float(ms), int(n))
    return out
