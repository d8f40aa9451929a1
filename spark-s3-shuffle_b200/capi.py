"""ctypes binding of include/b200shuffle.h — the same entry points the JNI shim binds (INTEGRATION.md §2).

Nothing here computes: every helper marshals numpy/bytes into plain pointers + sizes and calls libb200shuffle.so.
"""
import ctypes as C
import os

import numpy as np

from . import _build

# ---- constants mirrored from b200shuffle.h ----
CODEC_NONE, CODEC_LZ4BLOCK, CODEC_SNAPPY_XERIAL, CODEC_ZSTD = 0, 1, 2, 3
CHECKSUM_NONE, CHECKSUM_ADLER32, CHECKSUM_CRC32, CHECKSUM_CRC32C = 0, 1, 2, 3
KEY_BYTES, KEY_INT32, KEY_INT64 = 0, 1, 2  # key types of the row sort (decompress_sort_rows_*)
STRING_KEY = 3  # the composite-key calls' variable-length key column (decompress_*_rows_keys_*)
# the composite-key calls' other column types (BooleanType is KEY_BYTES with length 1) and order flags
KEY_INT16, KEY_INT8, KEY_FLOAT32, KEY_FLOAT64, DECIMAL_KEY = 5, 6, 7, 8, 9
KEY_DESCENDING, KEY_NULLS_LAST = 1 << 8, 1 << 9
# a null-safe (<=>) column, the pair (coalesce(v, default), isnull(v)): the join and hash calls only
KEY_NULL_SAFE = 1 << 10
# aggregate ops of the row aggregation (decompress_aggregate_rows_*)
(AGG_SUM_INT64, AGG_SUM_FLOAT64, AGG_MIN_INT32, AGG_MAX_INT32, AGG_MIN_INT64, AGG_MAX_INT64, AGG_MIN_FLOAT64,
 AGG_MAX_FLOAT64) = range(8)
# the Decimal ops (8 is unassigned); SUM_DECIMAL takes its buffer's precision P (1..38) as AGG_SUM_DECIMAL | P << 8
AGG_SUM_DECIMAL, AGG_MIN_DECIMAL, AGG_MAX_DECIMAL = 9, 10, 11
# Spark's CentralMomentAgg buffers [n, avg, m2] (stddev_*, var_*): one entry over three 8-byte doubles at off, off + 8,
# off + 16; never null (null field -1)
AGG_VARIANCE = 12
# join types of the row join (decompress_join_rows_keys_*) and the field kinds of its sides' schemas
JOIN_INNER, JOIN_LEFT_OUTER, JOIN_LEFT_SEMI, JOIN_LEFT_ANTI = 0, 1, 2, 3
JOIN_RIGHT_OUTER, JOIN_FULL_OUTER = 5, 6  # 4 is not assigned
JOIN_EXISTENCE = 8  # 7 is not assigned
FIELD_FIXED, FIELD_VAR, FIELD_DECIMAL_WIDE = 0, 1, 2
# ranking functions of the row window (decompress_window_rows_keys_*), and its limit function meaning "no limit"
WINDOW_ROW_NUMBER, WINDOW_RANK, WINDOW_DENSE_RANK, WINDOW_PERCENT_RANK, WINDOW_CUME_DIST, WINDOW_NTILE = range(6)
WINDOW_NO_LIMIT = 0xFFFFFFFF
# aggregate functions, frames and input types of the aggregate window (decompress_window_aggregate_rows_keys_*); a
# decimal(p, s) input is WINDOW_VAL_DECIMAL | p << 8 | s << 16 (window_val_decimal)
WINDOW_SUM, WINDOW_COUNT, WINDOW_MIN, WINDOW_MAX, WINDOW_AVG = range(6, 11)
WINDOW_FRAME_PARTITION, WINDOW_FRAME_ROWS_RUNNING, WINDOW_FRAME_RANGE_RUNNING = 1, 2, 3
(WINDOW_VAL_NONE, WINDOW_VAL_INT8, WINDOW_VAL_INT16, WINDOW_VAL_INT32, WINDOW_VAL_INT64, WINDOW_VAL_FLOAT32,
 WINDOW_VAL_FLOAT64, WINDOW_VAL_DECIMAL) = range(8)


# offset functions of the offset window (decompress_window_offset_rows_keys_*), its string / binary input type, and the
# per-function flags
WINDOW_LAG, WINDOW_LEAD, WINDOW_FIRST, WINDOW_LAST, WINDOW_NTH_VALUE = range(11, 16)
WINDOW_VAL_BYTES = 8
# the partial aggregation's central-moment function (aggregate_*partition_compress_rows_hash_*; its buffers n, avg and
# m2 are three partial-row fields, merged by AGG_VARIANCE); the window calls reject it
WINDOW_VARIANCE = 16
WINDOW_IGNORE_NULLS, WINDOW_HAS_DEFAULT = 1, 2
# the sliding frames of the frame window (decompress_window_frame_rows_keys_*) and their unbounded ends; a bound is
# otherwise 0 (CURRENT ROW), -k (k PRECEDING) or +k (k FOLLOWING)
WINDOW_FRAME_ROWS, WINDOW_FRAME_RANGE = 4, 5
WINDOW_UNBOUNDED_PRECEDING, WINDOW_UNBOUNDED_FOLLOWING = -2**63, 2**63 - 1


def window_val_decimal(p, s):
    return WINDOW_VAL_DECIMAL | p << 8 | s << 16
OK, E_CORRUPT, E_CHECKSUM, E_DST_TOO_SMALL, E_UNSUPPORTED, E_ARG, E_CUDA, E_NOT_INIT, E_NOMEM, E_NOT_CACHED = (
    0, -1, -2, -3, -4, -5, -6, -7, -8, -9)
NOT_RESIDENT = 2**64 - 1  # b2s_exchange_lookup's length of a map output that is not resident
CODEC_BY_NAME = {"lz4": CODEC_LZ4BLOCK, "snappy": CODEC_SNAPPY_XERIAL, "zstd": CODEC_ZSTD}
CHECKSUM_BY_NAME = {"ADLER32": CHECKSUM_ADLER32, "CRC32": CHECKSUM_CRC32, "CRC32C": CHECKSUM_CRC32C}


def agg_sum_decimal(precision):
    """the op of a Decimal(precision) sum buffer"""
    return AGG_SUM_DECIMAL | (precision << 8)


_u8p, _u64p, _u32p, _i32p, _vp = C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
_u32, _u64, _i32 = C.c_uint32, C.c_uint64, C.c_int32


class Timing(C.Structure):
    _fields_ = [
        ("total_ms", C.c_double), ("h2d_ms", C.c_double), ("d2h_ms", C.c_double), ("kernel_ms", C.c_double),
        ("top_kernel_ms", C.c_double), ("h2d_bytes", _u64), ("d2h_bytes", _u64), ("kernel_launches", _u64),
        ("src_bytes", _u64), ("dst_bytes", _u64), ("dominant_ms", C.c_double), ("dominant_launches", _u64),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# every symbol include/b200shuffle.h declares: (name, restype, argtypes)
PROTOTYPES = [
    ("b2s_init", C.c_int, [_u32, _u64, _u32]),
    ("b2s_shutdown", None, []),
    ("b2s_device_count", C.c_int, []),
    ("b2s_set_thread_device", C.c_int, [_u32]),
    ("b2s_bind_thread_to_device", C.c_int, [_u32]),
    ("b2s_device_numa_node", C.c_int, [_u32]),
    ("b2s_strerror", C.c_char_p, [_i32]),
    ("b2s_last_error", C.c_char_p, []),
    ("b2s_version", _u32, []),
    ("b2s_host_alloc", C.c_void_p, [_u64]),
    ("b2s_host_free", None, [C.c_void_p]),
    ("b2s_host_register", C.c_int, [C.c_void_p, _u64]),
    ("b2s_host_unregister", C.c_int, [C.c_void_p]),
    ("b2s_compress_bound", _u64, [_u32, _u32, _u64]),
    ("b2s_decompressed_size_batch", C.c_int, [_u32, _u32, _vp, _u64p, _u64p, _i32p]),
    ("b2s_checksum_batch", C.c_int, [_u32, _u32, _vp, _u64p, _u64p]),
    ("b2s_checksum_packed", C.c_int, [_u32, _u32, _u8p, _u64p, _u64p, _u64p]),
    ("b2s_compress_batch", C.c_int, [_u32, _i32, _u32, _u32, _u32, _vp, _u64p, _vp, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_compress_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_bound", _u64, [_u32, _u32, _u32, _u64]),
    ("b2s_partition_compress_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _u64, _vp, _u64, _u32p, _u32p, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_rows_hash_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u8p, _u64, _u64p,
      _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_rows_hash_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _u64, _vp, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _vp, _u64, _u64p,
      _u64p, _u64p, _u64p, _i32p]),
    ("b2s_aggregate_partition_compress_rows_hash_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u32p, _u32p, _u32p,
      _i32p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p]),
    ("b2s_aggregate_partition_compress_rows_hash_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _u64, _vp, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u32p, _u32p,
      _u32p, _i32p, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p]),
    ("b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u32p, _u32p, _u32p,
      _i32p, _u32, _u32p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p]),
    ("b2s_aggregate_grouping_sets_partition_compress_rows_hash_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _u64, _vp, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u32p, _u32p,
      _u32p, _i32p, _u32, _u32p, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p]),
    ("b2s_decompress_aggregate_distinct_partition_compress_rows_hash_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32, _u32p,
      _u32p, _u32, _u32p, _u32p, _i32p, _u32, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_aggregate_distinct_partition_compress_rows_hash_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32,
      _u32p, _u32p, _u32, _u32p, _u32p, _i32p, _u32, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p, _i32p,
      _i32p]),
    ("b2s_window_limit_partition_compress_rows_hash_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _i32, _u8p,
      _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p]),
    ("b2s_window_limit_partition_compress_rows_hash_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _u64, _vp, _u64, _u32p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _i32,
      _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _u64p]),
    ("b2s_partition_compress_rows_range_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u8p, _u64, _u32p,
      _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_rows_range_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u64, _vp, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u8p, _u64, _u32p,
      _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_rows_round_robin_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _i32, _u32, _u64, _u8p, _u64, _u32p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p,
      _i32p]),
    ("b2s_partition_compress_rows_round_robin_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _i32, _u32, _u64, _vp, _u64, _u32p, _vp, _u64, _u64p, _u64p, _u64p, _u64p,
      _i32p]),
    ("b2s_decompress_batch", C.c_int,
     [_u32, _u32, _u32, _vp, _u64p, _u32p, _vp, _vp, _vp, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_sort_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _u8p, _u64, _u64p, _u64p, _i32p,
      _i32p]),
    ("b2s_decompress_sort_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _vp, _u64, _u64p, _u64p, _i32p,
      _i32p]),
    ("b2s_decompress_sort_rows_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _i32, _u8p, _u64, _u64p, _u64p,
      _i32p, _i32p]),
    ("b2s_decompress_sort_rows_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _i32, _vp, _u64, _u64p, _u64p,
      _i32p, _i32p]),
    ("b2s_decompress_aggregate_rows_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _i32, _u32, _u32p, _u32p, _i32p,
      _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_aggregate_rows_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _i32, _u32, _u32p, _u32p, _i32p,
      _vp, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_sort_rows_keys_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p, _i32p, _u8p, _u64, _u64p,
      _u64p, _i32p, _i32p]),
    ("b2s_decompress_sort_rows_keys_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p, _i32p, _vp, _u64,
      _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_aggregate_rows_keys_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u32p, _u32p,
      _i32p, _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_aggregate_rows_keys_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u32p,
      _u32p, _i32p, _vp, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_join_rows_keys_packed", C.c_int,
     [_u32, _u32, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p, _i32p, _u32p,
      _i32p, _u32, _u8p, _u32, _u8p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_join_rows_keys_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p, _i32p,
      _u32p, _i32p, _u32, _u8p, _u32, _u8p, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_window_rows_keys_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u8p,
      _u32, _u32p, _i32p, _u32, _i32, _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_window_rows_keys_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32,
      _u8p, _u32, _u32p, _i32p, _u32, _i32, _vp, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_window_aggregate_rows_keys_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u8p,
      _u32, _u32p, _i32p, _u32p, _u32p, _u32p, _i32p, _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_window_aggregate_rows_keys_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32,
      _u8p, _u32, _u32p, _i32p, _u32p, _u32p, _u32p, _i32p, _vp, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_window_offset_rows_keys_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u8p,
      _u32, _u32p, _i32p, _u32p, _u32p, _u32p, _i32p, _u32p, _u64p, _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_window_offset_rows_keys_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32,
      _u8p, _u32, _u32p, _i32p, _u32p, _u32p, _u32p, _i32p, _u32p, _u64p, _vp, _u64, _u64p, _u64p, _u64p, _i32p,
      _i32p]),
    ("b2s_decompress_window_frame_rows_keys_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u8p,
      _u32, _u32p, _i32p, _u32p, _u32p, _u32p, _i32p, _u32p, _u64p, _vp, _vp, _u8p, _u64, _u64p, _u64p, _u64p, _i32p,
      _i32p]),
    ("b2s_decompress_window_frame_rows_keys_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32p, _u32p, _u32p, _i32p, _u32,
      _u8p, _u32, _u32p, _i32p, _u32p, _u32p, _u32p, _i32p, _u32p, _u64p, _vp, _vp, _vp, _u64, _u64p, _u64p, _u64p,
      _i32p, _i32p]),
    ("b2s_exchange_set_budget", C.c_int, [_u32, _u64]),
    ("b2s_partition_compress_cached_packed", C.c_int,
     [_i32, C.c_int64, _u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32p, _u8p, _u64, _u64p, _u64p, _u64p,
      _u64p, _i32p, _i32p]),
    ("b2s_exchange_lookup", C.c_int, [_i32, _i32, _i32, _u32, _vp, _u64p]),
    ("b2s_exchange_read_packed", C.c_int, [_i32, _i32, _i32, _u32, _vp, _u8p, _u64, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_exchange_read_sort_packed", C.c_int,
     [_i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _u8p,
      _u64, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_read_sort_dev", C.c_int,
     [_u32, _i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32,
      _vp, _u64, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_partition_compress_rows_hash_cached_packed", C.c_int,
     [_i32, C.c_int64, _u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u8p,
      _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_partition_compress_rows_range_cached_packed", C.c_int,
     [_i32, C.c_int64, _u32, _i32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32, _u32p, _u32p, _u32p, _i32p, _u32, _u8p,
      _u64, _u32p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_partition_compress_rows_round_robin_cached_packed", C.c_int,
     [_i32, C.c_int64, _u32, _i32, _u32, _u32, _u32, _i32, _u32, _u64, _u8p, _u64, _u32p, _u8p, _u64, _u64p, _u64p,
      _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_read_sort_rows_keys_packed", C.c_int,
     [_i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p,
      _i32p, _u8p, _u64, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_read_sort_rows_keys_dev", C.c_int,
     [_u32, _i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p,
      _u32p, _i32p, _vp, _u64, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_read_aggregate_rows_keys_packed", C.c_int,
     [_i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p, _u32p,
      _i32p, _u32, _u32p, _u32p, _i32p, _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_read_aggregate_rows_keys_dev", C.c_int,
     [_u32, _i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32p, _u32p,
      _u32p, _i32p, _u32, _u32p, _u32p, _i32p, _vp, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_remove", C.c_int, [_i32, C.c_int64]),
    ("b2s_checksum_dev", C.c_int, [_u32, _u32, _u32, _vp, _u64p, _u64p, _u64p]),
    ("b2s_compress_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _vp, _u64p, _u64p, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_decompress_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _vp, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_dev_alloc", C.c_void_p, [_u32, _u64]),
    ("b2s_dev_free", None, [_u32, C.c_void_p]),
    ("b2s_dev_memcpy", C.c_int, [_u32, C.c_void_p, C.c_void_p, _u64, C.c_int]),
    ("b2s_last_timing", C.c_int, [C.POINTER(Timing)]),
    ("b2s_total_kernel_launches", _u64, []),
    ("b2s_mark", C.c_int, [_u32, _u32]),
    ("b2s_marks_elapsed_ms", C.c_int, [_u32, C.POINTER(C.c_double)]),
    ("b2s_gen_terasort_dev", C.c_int, [_u32, C.c_void_p, _u64, _u64, _u64]),
]
SYMBOLS = [p[0] for p in PROTOTYPES]

_lib = None


def load(build_if_needed=True):
    """Loads libb200shuffle.so (building it with nvcc when stale).  Raises if that is impossible — no fallback."""
    global _lib
    if _lib is None:
        path = _build.build() if build_if_needed else _build.LIB
        if not os.path.exists(path):
            raise RuntimeError("libb200shuffle.so is missing and could not be built; there is no CPU fallback")
        L = C.CDLL(path)
        for name, res, args in PROTOTYPES:
            f = getattr(L, name)  # AttributeError if the library does not export a declared symbol
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


class B2SError(RuntimeError):
    def __init__(self, code, where):
        L = load()
        self.code = code
        msg = L.b2s_strerror(code).decode()
        detail = L.b2s_last_error().decode()
        super().__init__("%s: %s (%d)%s" % (where, msg, code, (": " + detail) if detail else ""))


def _check(rc, where):
    if rc != 0:
        raise B2SError(rc, where)


def init(gpu_mask=0, pinned_bytes_per_gpu=0, streams_per_gpu=0):
    _check(load().b2s_init(gpu_mask, pinned_bytes_per_gpu, streams_per_gpu), "b2s_init")


def bind_thread_to_device(dev=0):
    """pins the calling thread to the CPUs of the device's NUMA node and prefers that node for its allocations"""
    _check(load().b2s_bind_thread_to_device(dev), "b2s_bind_thread_to_device")
    return load().b2s_device_numa_node(dev)


def shutdown():
    load().b2s_shutdown()


def last_timing():
    t = Timing()
    load().b2s_last_timing(C.byref(t))
    return t.as_dict()


def mark(which, dev=0):
    _check(load().b2s_mark(dev, which), "b2s_mark")


def marks_elapsed_ms(dev=0):
    ms = C.c_double(0)
    _check(load().b2s_marks_elapsed_ms(dev, C.byref(ms)), "b2s_marks_elapsed_ms")
    return ms.value


def compress_bound(codec, block_size, n):
    return load().b2s_compress_bound(codec, block_size, n)


# ---------------------------------------------------------------------------------------------------------------
# marshalling helpers
# ---------------------------------------------------------------------------------------------------------------
def _as_u8(b):
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b, dtype=np.uint8)
    return np.frombuffer(b, dtype=np.uint8)


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def _ptr_array(arrs):
    out = np.zeros(max(len(arrs), 1), dtype=np.uint64)
    for i, a in enumerate(arrs):
        out[i] = a.ctypes.data if a.size else 0
    return out


class HostBuffer:
    """Pinned host memory from b2s_host_alloc, viewed as a numpy uint8 array (what the JVM wraps as a direct buffer)."""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        self.ptr = load().b2s_host_alloc(max(self.nbytes, 1))
        if not self.ptr:
            raise B2SError(E_NOMEM, "b2s_host_alloc")
        buf = (C.c_uint8 * max(self.nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=np.uint8, count=self.nbytes)

    def free(self):
        if self.ptr:
            self.array = None
            load().b2s_host_free(self.ptr)
            self.ptr = None


# ---------------------------------------------------------------------------------------------------------------
# host-pointer API
# ---------------------------------------------------------------------------------------------------------------
def checksum_batch(alg, blocks):
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    ptrs = _ptr_array(arrs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    out = np.zeros(max(n, 1), dtype=np.uint64)
    _check(load().b2s_checksum_batch(alg, n, _ptr(ptrs), _ptr(lens), _ptr(out)), "b2s_checksum_batch")
    return [int(v) for v in out[:n]]


def checksum_packed(alg, base, off, length):
    base = _as_u8(base)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    out = np.zeros(max(off.size, 1), dtype=np.uint64)
    _check(load().b2s_checksum_packed(alg, off.size, _ptr(base), _ptr(off), _ptr(length), _ptr(out)),
           "b2s_checksum_packed")
    return out[: off.size]


def compress_batch(codec, blocks, block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dst_caps=None):
    """-> (list of compressed streams (bytes or None on error), checksums, status)"""
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    caps = np.array(
        (dst_caps if dst_caps is not None else [compress_bound(codec, block_size, a.size) for a in arrs]) or [0],
        dtype=np.uint64)
    outs = [np.empty(int(c), dtype=np.uint8) for c in caps[:n]]
    sp, dp = _ptr_array(arrs), _ptr_array(outs)
    dlen = np.zeros(max(n, 1), dtype=np.uint64)
    cks = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    _check(load().b2s_compress_batch(codec, level, block_size, checksum_alg, n, _ptr(sp), _ptr(lens), _ptr(dp),
                                     _ptr(caps), _ptr(dlen), _ptr(cks), _ptr(st)), "b2s_compress_batch")
    res = [outs[i][: int(dlen[i])].tobytes() if st[i] == 0 else None for i in range(n)]
    return res, [int(v) for v in cks[:n]], [int(v) for v in st[:n]]


def compress_packed(codec, src, off, length, dst, block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """src/dst: uint8 arrays (ideally HostBuffer.array).  -> dict(dst_off, dst_len, total, checksums, status)"""
    src, dst = _as_u8(src), _as_u8(dst)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    cks = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_compress_packed(codec, level, block_size, checksum_alg, n, _ptr(src), _ptr(off), _ptr(length),
                                      _ptr(dst), dst.size, _ptr(dst_off), _ptr(dst_len), C.addressof(total),
                                      _ptr(cks), _ptr(st)), "b2s_compress_packed")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, checksums=cks[:n], status=st[:n])


def partition_compress_bound(codec, block_size, num_partitions, rec_bytes):
    return load().b2s_partition_compress_bound(codec, block_size, num_partitions, rec_bytes)


def _partition_out(num_partitions):
    return (np.zeros(num_partitions, dtype=np.uint64), np.zeros(num_partitions, dtype=np.uint64),
            np.zeros(num_partitions, dtype=np.uint64), np.zeros(num_partitions, dtype=np.int32))


def _records(records, rec_len):
    """a packed call's records (back to back) and their lengths -> its arguments n_records, rec_base, rec_bytes,
    rec_len"""
    records, rec_len = _as_u8(records), np.ascontiguousarray(rec_len, dtype=np.uint32)
    return rec_len.size, records, records.size, rec_len


def _partition_call(symbol, codec, level, block_size, checksum_alg, num_partitions, mid, dst, dst_cap=None, dev=None,
                    lead=(), counts=()):
    """One map-side partition call, whose arguments are [dev,] *lead, codec, level, block_size, checksum_alg, *mid, dst,
    dst_cap, dst_off, dst_len, total, checksums, status, *counts.  dev None: the packed form, dst a host array (dst_cap
    is its size); else dst is a device address.  lead and mid are the call's own arguments, numpy arrays among them
    passed as pointers (_records gives a packed call's records); counts names the outputs after status (n_groups,
    n_out_records or cached).  -> dict(dst_off, dst_len, total, checksums, status, *counts)"""
    if dev is None:
        dst = _as_u8(dst)
        dst_cap = dst.size
    dst_off, dst_len, cks, st = _partition_out(num_partitions)
    total = _u64(0)
    outs = [_i32(0) if name == "cached" else _u64(0) for name in counts]
    args = ([] if dev is None else [dev]) + [*lead, codec, level, block_size, checksum_alg, *mid, dst, dst_cap]
    _check(getattr(load(), symbol)(*map(_arg, args), _ptr(dst_off), _ptr(dst_len), C.addressof(total), _ptr(cks),
                                   _ptr(st), *map(C.addressof, outs)), symbol)
    r = dict(dst_off=dst_off, dst_len=dst_len, total=total.value, checksums=cks, status=st)
    r.update(zip(counts, (o.value for o in outs)))
    return r


def partition_compress_packed(codec, records, rec_len, rec_part, num_partitions, dst, block_size=0,
                              checksum_alg=CHECKSUM_NONE, level=0):
    """records: the serialized records back to back (uint8 array, ideally HostBuffer.array); rec_len / rec_part: one
    length and one reduce id per record.  -> dict(dst_off, dst_len, total, checksums, status), one entry per partition"""
    return _partition_call("b2s_partition_compress_packed", codec, level, block_size, checksum_alg, num_partitions,
                           (num_partitions, *_records(records, rec_len), np.ascontiguousarray(rec_part, np.uint32)),
                           dst)


def decompressed_size_batch(codec, blocks):
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    sp = _ptr_array(arrs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    out = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    _check(load().b2s_decompressed_size_batch(codec, n, _ptr(sp), _ptr(lens), _ptr(out), _ptr(st)),
           "b2s_decompressed_size_batch")
    return [int(v) for v in out[:n]], [int(v) for v in st[:n]]


def decompress_batch(codec, blocks, checksum_alg=CHECKSUM_NONE, slices=None, dst_caps=None):
    """slices: per block a list of (length, checksum) pairs (the block's .index differences / .checksum values).
    -> (list of decoded bytes or None, status, bad_slice)"""
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    if dst_caps is None:
        sizes, _ = decompressed_size_batch(codec, blocks)
        dst_caps = sizes
    caps = np.array(list(dst_caps) or [0], dtype=np.uint64)
    outs = [np.empty(max(int(c), 1), dtype=np.uint8) for c in caps[:n]]
    sp, dp = _ptr_array(arrs), _ptr_array(outs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    dlen = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    ns = sl_ptrs = sc_ptrs = None
    keep = []
    if checksum_alg != CHECKSUM_NONE:
        ns = np.array([len(s) for s in slices] or [0], dtype=np.uint32)
        sl = [np.array([p[0] for p in s] or [0], dtype=np.uint64) for s in slices]
        sc = [np.array([p[1] for p in s] or [0], dtype=np.uint64) for s in slices]
        keep = [sl, sc]
        sl_ptrs = np.array([a.ctypes.data for a in sl] or [0], dtype=np.uint64)
        sc_ptrs = np.array([a.ctypes.data for a in sc] or [0], dtype=np.uint64)
    _check(load().b2s_decompress_batch(codec, checksum_alg, n, _ptr(sp), _ptr(lens), _ptr(ns), _ptr(sl_ptrs),
                                       _ptr(sc_ptrs), _ptr(dp), _ptr(caps), _ptr(dlen), _ptr(st), _ptr(bad)),
           "b2s_decompress_batch")
    del keep
    res = [outs[i][: int(dlen[i])].tobytes() if st[i] == 0 else None for i in range(n)]
    return res, [int(v) for v in st[:n]], [int(v) for v in bad[:n]]


def _slice_arrays(checksum_alg, slice_base, slice_len, slice_checksum):
    if checksum_alg == CHECKSUM_NONE:
        return None, None, None
    return (np.ascontiguousarray(slice_base, dtype=np.uint32), np.ascontiguousarray(slice_len, dtype=np.uint64),
            np.ascontiguousarray(slice_checksum, dtype=np.uint64))


def decompress_packed(codec, src, off, length, dst, checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                      slice_checksum=None):
    src, dst = _as_u8(src), _as_u8(dst)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    sb, sl, sc = _slice_arrays(checksum_alg, slice_base, slice_len, slice_checksum)
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_decompress_packed(codec, checksum_alg, n, _ptr(src), _ptr(off), _ptr(length), _ptr(sb), _ptr(sl),
                                        _ptr(sc), _ptr(dst), dst.size, _ptr(dst_off), _ptr(dst_len),
                                        C.addressof(total), _ptr(st), _ptr(bad)), "b2s_decompress_packed")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, status=st[:n], bad_slice=bad[:n])


def _agg_arrays(aggs):
    """aggs = [(op, off, null_field), ...] -> (n, op, off, null_field) arrays"""
    aggs = list(aggs)
    op = np.array([a[0] for a in aggs] or [0], dtype=np.uint32)
    off = np.array([a[1] for a in aggs] or [0], dtype=np.uint32)
    nf = np.array([a[2] for a in aggs] or [0], dtype=np.int32)
    return len(aggs), op, off, nf


def _key_arrays(keys):
    """keys = [(key_type, key_off, key_len, null_field), ...] -> (n, type, off, len, null_field) arrays"""
    keys = list(keys)
    kt = np.array([k[0] for k in keys] or [0], dtype=np.uint32)
    ko = np.array([k[1] for k in keys] or [0], dtype=np.uint32)
    kl = np.array([k[2] for k in keys] or [0], dtype=np.uint32)
    kn = np.array([k[3] for k in keys] or [0], dtype=np.int32)
    return len(keys), kt, ko, kl, kn


def _arg(a):
    return _ptr(a) if isinstance(a, np.ndarray) else a


def _sort_call(symbol, codec, src, off, length, dst, dst_cap, mid, checksum_alg, slices, dev=None, lead=(), n=None,
               before_n=()):
    """One call of the sort family, whose arguments are [dev,] *lead, codec, checksum_alg, *before_n, n, src, off,
    length, the three slice arrays, *mid, dst, dst_cap, total, n_records, [n_groups,] status, bad_slice.  dev None: the
    packed form, src and dst host arrays (dst_cap is dst's size); else src and dst are device addresses.  lead,
    before_n and mid are the call's own arguments, numpy arrays among them passed as pointers; n defaults to the number
    of blocks in off.  -> dict(total, n_records, status, bad_slice), with n_groups after n_records for the aggregate
    calls; the join calls return n_left_records, n_right_records and n_out_records in n_records' place, the window
    calls n_records and n_out_records"""
    if dev is None:
        src, dst = _as_u8(src), _as_u8(dst)
        dst_cap = dst.size
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size if n is None else n
    sb, sl, sc = _slice_arrays(checksum_alg, *slices)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    names = (("total", "n_left_records", "n_right_records", "n_out_records") if "_join_" in symbol else
             ("total", "n_records", "n_out_records") if "_window_" in symbol else
             ("total", "n_records", "n_groups") if "_aggregate_" in symbol else ("total", "n_records"))
    counts = [_u64(0) for _ in names]
    args = ([] if dev is None else [dev]) + [*lead, codec, checksum_alg, *before_n, n, src, off, length, sb, sl, sc,
                                             *mid, dst, dst_cap]
    _check(getattr(load(), symbol)(*map(_arg, args), *map(C.addressof, counts), _ptr(st), _ptr(bad)), symbol)
    r = dict(zip(names, (c.value for c in counts)))
    r.update(status=st[:n], bad_slice=bad[:n])
    return r


def decompress_sort_packed(codec, src, off, length, dst, record_bytes, key_off, key_len, checksum_alg=CHECKSUM_NONE,
                           slice_base=None, slice_len=None, slice_checksum=None):
    """Verifies and decodes a reduce task's blocks and sorts their fixed-size records by the unsigned bytes
    [key_off, key_off + key_len) into dst (stable).  -> dict(total, n_records, status, bad_slice)"""
    return _sort_call("b2s_decompress_sort_packed", codec, src, off, length, dst, None,
                      (record_bytes, key_off, key_len), checksum_alg, (slice_base, slice_len, slice_checksum))


def decompress_sort_rows_packed(codec, src, off, length, dst, key_type, key_off, key_len, null_field=-1,
                                checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None, slice_checksum=None):
    """Verifies and decodes a reduce task's blocks of length-prefixed UnsafeRow records ([int32 big-endian size][row])
    and sorts the records by the typed key at row offset key_off (KEY_BYTES / KEY_INT32 / KEY_INT64; nulls first when
    null_field >= 0) into dst (stable).  -> dict(total, n_records, status, bad_slice)"""
    return _sort_call("b2s_decompress_sort_rows_packed", codec, src, off, length, dst, None,
                      (key_type, key_off, key_len, null_field), checksum_alg, (slice_base, slice_len, slice_checksum))


def decompress_aggregate_rows_packed(codec, src, off, length, dst, key_type, key_off, key_len, null_field=-1, aggs=(),
                                     checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None, slice_checksum=None):
    """Verifies and decodes a reduce task's blocks of UnsafeRow records, groups them by the typed key (as
    decompress_sort_rows_packed orders them) and merges every aggregate (op AGG_*, 8-byte slot at row offset off,
    null bit null_field or -1) over each group into one row per group in dst.
    -> dict(total, n_records, n_groups, status, bad_slice)"""
    return _sort_call("b2s_decompress_aggregate_rows_packed", codec, src, off, length, dst, None,
                      (key_type, key_off, key_len, null_field, *_agg_arrays(aggs)), checksum_alg,
                      (slice_base, slice_len, slice_checksum))


def decompress_sort_rows_keys_packed(codec, src, off, length, dst, keys, checksum_alg=CHECKSUM_NONE, slice_base=None,
                                     slice_len=None, slice_checksum=None):
    """decompress_sort_rows_packed by a composite key: keys = [(key type, row offset, length, null field or -1), ...],
    compared left to right.  A key type is KEY_BYTES (1..16 bytes), KEY_INT8 / INT16 / INT32 / INT64 (1 / 2 / 4 / 8),
    KEY_FLOAT32 / FLOAT64 (4 / 8, Spark SQL's order: -0.0 == 0.0, NaN above +inf), STRING_KEY or DECIMAL_KEY (the
    8-byte (offset << 32) | size slot of a string, or of a Decimal(p > 18)'s 1..16 big-endian bytes), OR-ed with
    KEY_DESCENDING (the column's values in reverse) and / or KEY_NULLS_LAST (its nulls after its values); without
    flags a column is ascending, nulls first.  -> dict(total, n_records, status, bad_slice)"""
    return _sort_call("b2s_decompress_sort_rows_keys_packed", codec, src, off, length, dst, None, _key_arrays(keys),
                      checksum_alg, (slice_base, slice_len, slice_checksum))


def decompress_aggregate_rows_keys_packed(codec, src, off, length, dst, keys, aggs=(), checksum_alg=CHECKSUM_NONE,
                                          slice_base=None, slice_len=None, slice_checksum=None):
    """decompress_aggregate_rows_packed grouped by a composite key (keys as in decompress_sort_rows_keys_packed; the
    groups come out in that order, and float keys group by Spark SQL's equality: 0.0 with -0.0, every NaN together).
    -> dict(total, n_records, n_groups, status, bad_slice)"""
    return _sort_call("b2s_decompress_aggregate_rows_keys_packed", codec, src, off, length, dst, None,
                      (*_key_arrays(keys), *_agg_arrays(aggs)), checksum_alg, (slice_base, slice_len, slice_checksum))


def _join_arrays(left_keys, right_keys, left_kinds, right_kinds):
    """the join's key and field-kind arguments: the columns' types and lengths are the left keys', each side's slots
    and null fields its own; a kinds sequence of None is passed as NULL"""
    n, kt, lo, kl, ln = _key_arrays(left_keys)
    _, _, ro, _, rn = _key_arrays(right_keys)
    kinds = [None if k is None else np.ascontiguousarray(k, dtype=np.uint8) for k in (left_kinds, right_kinds)]
    return n, kt, kl, lo, ln, ro, rn, kinds[0], kinds[1]


def decompress_join_rows_keys_packed(join_type, codec, src, off, length, n_left, dst, left_keys, right_keys,
                                     n_left_fields, n_right_fields, left_kinds=None, right_kinds=None,
                                     checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                     slice_checksum=None):
    """Sort-merge joins a reducer's two shuffled sides of UnsafeRow records: blocks [0, n_left) are the left side's,
    the rest the right's.  left_keys / right_keys: [(key type, row offset, length, null field or -1), ...] as in
    decompress_sort_rows_keys_packed without order flags, one entry per join key column on each side (the types and
    lengths are the left's); a type OR-ed with KEY_NULL_SAFE is a null-safe (<=>) column, equal to a null when null.
    The kinds (FIELD_*, one per field; None for semi and anti joins, and the right's for JOIN_EXISTENCE) say which slots
    hold an offset.  dst receives Spark's joined rows ([int32 big-endian size][row]) for JOIN_INNER / JOIN_LEFT_OUTER /
    JOIN_RIGHT_OUTER / JOIN_FULL_OUTER (left.output ++ right.output; a right outer join in the right side's key order,
    a full outer join run by run in key order, as the header states), the left records for JOIN_LEFT_SEMI /
    JOIN_LEFT_ANTI, and for JOIN_EXISTENCE every left record with one boolean field, whether it has a match
    (left.output :+ exists).
    -> dict(total, n_left_records, n_right_records, n_out_records, status, bad_slice)"""
    n, kt, kl, lo, ln, ro, rn, lk, rk = _join_arrays(left_keys, right_keys, left_kinds, right_kinds)
    return _sort_call("b2s_decompress_join_rows_keys_packed", codec, src, off, length, dst, None,
                      (n, kt, kl, lo, ln, ro, rn, n_left_fields, lk, n_right_fields, rk), checksum_alg,
                      (slice_base, slice_len, slice_checksum), lead=(join_type,), before_n=(n_left,))


def _window_arrays(keys, n_partition_keys, n_fields, kinds, fns, limit):
    """the window's key, field-kind, function and limit arguments: fns = [fn or (WINDOW_NTILE, k), ...]; limit None
    (no limit) or (limit_fn, limit)"""
    n, kt, ko, kl, kn = _key_arrays(keys)
    fns = [f if isinstance(f, tuple) else (f, 0) for f in fns]
    fn = np.array([f[0] for f in fns] or [0], dtype=np.uint32)
    arg = np.array([f[1] for f in fns] or [0], dtype=np.int32)
    kinds = None if kinds is None else np.ascontiguousarray(kinds, dtype=np.uint8)
    limit_fn, lim = (WINDOW_NO_LIMIT, 0) if limit is None else limit
    return n_partition_keys, n, kt, ko, kl, kn, n_fields, kinds, len(fns), fn, arg, limit_fn, lim


def _window_fn_rows(fns):
    """fns -> [(fn, arg, frame, val_type, val_off, val_null_field, flags, default)]: a ranking fn or (WINDOW_NTILE, k),
    an aggregate (fn, frame, val_type, val_off, val_null_field), or an offset function in the full form"""
    full = []
    for f in fns:
        if isinstance(f, tuple) and len(f) == 8:
            full.append(tuple(f))
        elif isinstance(f, tuple) and len(f) == 5:
            full.append((f[0], 0) + tuple(f[1:]) + (0, 0))
        else:
            fn, arg = f if isinstance(f, tuple) else (f, 0)
            full.append((fn, arg, 0, WINDOW_VAL_NONE, 0, -1, 0, 0))
    return full


def _window_aggregate_arrays(keys, n_partition_keys, n_fields, kinds, fns, offset=False):
    """the aggregate window's key, field-kind and function arguments: fns = [ranking fn, (WINDOW_NTILE, k), or an
    aggregate (fn, frame, val_type, val_off, val_null_field)]; offset: the offset window's, whose fns may also be
    offset functions (fn, arg, frame, val_type, val_off, val_null_field, flags, default), with the flags and defaults"""
    n, kt, ko, kl, kn = _key_arrays(keys)
    full = _window_fn_rows(fns)
    cols = list(zip(*full)) if full else [[0]] * 8
    fn, arg, frame, vt, vo, vn, fl, dv = (np.array(c, dtype=t) for c, t in zip(cols, (
        np.uint32, np.int32, np.uint32, np.uint32, np.uint32, np.int32, np.uint32, np.uint64)))
    kinds = None if kinds is None else np.ascontiguousarray(kinds, dtype=np.uint8)
    a = (n_partition_keys, n, kt, ko, kl, kn, n_fields, kinds, len(full), fn, arg, frame, vt, vo, vn)
    return a + (fl, dv) if offset else a


def _window_offset_arrays(keys, n_partition_keys, n_fields, kinds, fns):
    return _window_aggregate_arrays(keys, n_partition_keys, n_fields, kinds, fns, offset=True)


def _window_frame_arrays(keys, n_partition_keys, n_fields, kinds, fns):
    """the frame window's arguments: the offset window's, fns also taking (fn, arg, frame, val_type, val_off,
    val_null_field, flags, default, lower, upper) (every other form has bounds 0), with the bounds appended"""
    bounds = [tuple(f[8:]) if isinstance(f, tuple) and len(f) == 10 else (0, 0) for f in fns]
    rows = [tuple(f[:8]) if isinstance(f, tuple) and len(f) == 10 else f for f in fns]
    lo, hi = (np.array([b[u] for b in bounds] or [0], dtype=np.int64) for u in (0, 1))
    return _window_aggregate_arrays(keys, n_partition_keys, n_fields, kinds, rows, offset=True) + (lo, hi)


def decompress_window_frame_rows_keys_packed(codec, src, off, length, dst, keys, n_partition_keys, n_fields, kinds, fns,
                                             checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                             slice_checksum=None):
    """Spark's WindowExec over sliding ROWS and RANGE frames (with ranking, offset and aggregate functions) over a
    reducer's UnsafeRow records: as decompress_window_offset_rows_keys_packed, fns also taking (fn, arg, frame,
    val_type, val_off, val_null_field, flags, default, lower, upper) with frame WINDOW_FRAME_ROWS or WINDOW_FRAME_RANGE
    and the bounds WINDOW_UNBOUNDED_PRECEDING / WINDOW_UNBOUNDED_FOLLOWING, 0 (CURRENT ROW), -k or +k.
    -> dict(total, n_records, n_out_records, status, bad_slice)"""
    return _sort_call("b2s_decompress_window_frame_rows_keys_packed", codec, src, off, length, dst, None,
                      _window_frame_arrays(keys, n_partition_keys, n_fields, kinds, fns), checksum_alg,
                      (slice_base, slice_len, slice_checksum))


def decompress_window_offset_rows_keys_packed(codec, src, off, length, dst, keys, n_partition_keys, n_fields, kinds,
                                              fns, checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                              slice_checksum=None):
    """Spark's WindowExec with offset (and ranking and aggregate) functions over a reducer's UnsafeRow records: as
    decompress_window_aggregate_rows_keys_packed, fns also taking offset functions (WINDOW_LAG / LEAD / FIRST / LAST /
    NTH_VALUE, its offset or n (0 for FIRST and LAST), its frame (0 for LAG and LEAD), WINDOW_VAL_* (WINDOW_VAL_BYTES for
    a string or binary), window_val_decimal(p, s), the input's slot offset, its null bit or -1, WINDOW_IGNORE_NULLS |
    WINDOW_HAS_DEFAULT, the default's slot bits).  A string value's bytes follow the input's var bytes, padded to 8.
    -> dict(total, n_records, n_out_records, status, bad_slice)"""
    return _sort_call("b2s_decompress_window_offset_rows_keys_packed", codec, src, off, length, dst, None,
                      _window_offset_arrays(keys, n_partition_keys, n_fields, kinds, fns), checksum_alg,
                      (slice_base, slice_len, slice_checksum))


def decompress_window_aggregate_rows_keys_packed(codec, src, off, length, dst, keys, n_partition_keys, n_fields,
                                                 kinds, fns, checksum_alg=CHECKSUM_NONE, slice_base=None,
                                                 slice_len=None, slice_checksum=None):
    """Spark's WindowExec with aggregate (and ranking) functions over a reducer's UnsafeRow records: as
    decompress_window_rows_keys_packed without a limit, fns mixing ranking functions (as there) and aggregates
    (WINDOW_SUM / COUNT / MIN / MAX / AVG, WINDOW_FRAME_*, WINDOW_VAL_* or window_val_decimal(p, s), the input's slot
    offset, its null bit or -1).  An aggregate's value is null when its frame has no input, and a decimal result above
    precision 18 takes 16 bytes after the input's var bytes.  -> dict(total, n_records, n_out_records, status,
    bad_slice)"""
    return _sort_call("b2s_decompress_window_aggregate_rows_keys_packed", codec, src, off, length, dst, None,
                      _window_aggregate_arrays(keys, n_partition_keys, n_fields, kinds, fns), checksum_alg,
                      (slice_base, slice_len, slice_checksum))


def decompress_window_rows_keys_packed(codec, src, off, length, dst, keys, n_partition_keys, n_fields, kinds, fns,
                                       limit=None, checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                       slice_checksum=None):
    """Spark's WindowExec with ranking functions over a reducer's UnsafeRow records: keys as in
    decompress_sort_rows_keys_packed, the first n_partition_keys of them the PARTITION BY columns (no order flags), the
    rest the ORDER BY columns; n_fields / kinds (FIELD_*, one per field) the input schema; fns the functions
    (WINDOW_ROW_NUMBER, WINDOW_RANK, WINDOW_DENSE_RANK, WINDOW_PERCENT_RANK, WINDOW_CUME_DIST, or (WINDOW_NTILE, k)),
    each appended to the row as one 8-byte field; limit None or (WINDOW_ROW_NUMBER / RANK / DENSE_RANK, n): only the
    rows whose value of that function is at most n (WindowGroupLimitExec).  dst receives the output rows in sorted
    order ([int32 big-endian size][row], the input row joined with the values as UnsafeRowJoiner joins them).
    -> dict(total, n_records, n_out_records, status, bad_slice)"""
    return _sort_call("b2s_decompress_window_rows_keys_packed", codec, src, off, length, dst, None,
                      _window_arrays(keys, n_partition_keys, n_fields, kinds, fns, limit), checksum_alg,
                      (slice_base, slice_len, slice_checksum))


# ---------------------------------------------------------------------------------------------------------------
# device-resident API (bench.py roofline leg); d_* are raw device addresses (ints)
# ---------------------------------------------------------------------------------------------------------------
def dev_alloc(nbytes, dev=0):
    p = load().b2s_dev_alloc(dev, nbytes)
    if not p:
        raise B2SError(E_NOMEM, "b2s_dev_alloc")
    return p


def dev_free(p, dev=0):
    load().b2s_dev_free(dev, p)


def dev_memcpy(dst, src, nbytes, kind, dev=0):
    _check(load().b2s_dev_memcpy(dev, dst, src, nbytes, kind), "b2s_dev_memcpy")


def gen_terasort_dev(d_dst, first_record, n_records, seed=42, dev=0):
    _check(load().b2s_gen_terasort_dev(dev, d_dst, first_record, n_records, seed), "b2s_gen_terasort_dev")


def checksum_dev(alg, d_base, off, length, dev=0):
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    out = np.zeros(max(off.size, 1), dtype=np.uint64)
    _check(load().b2s_checksum_dev(dev, alg, off.size, d_base, _ptr(off), _ptr(length), _ptr(out)), "b2s_checksum_dev")
    return out[: off.size]


def compress_dev(codec, d_src, off, length, d_dst, dst_cap, block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    cks = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_compress_dev(dev, codec, level, block_size, checksum_alg, n, d_src, _ptr(off), _ptr(length),
                                   d_dst, dst_cap, _ptr(dst_off), _ptr(dst_len), C.addressof(total), _ptr(cks),
                                   _ptr(st)), "b2s_compress_dev")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, checksums=cks[:n], status=st[:n])


def decompress_dev(codec, d_src, off, length, d_dst, dst_cap, checksum_alg=CHECKSUM_NONE, slice_base=None,
                   slice_len=None, slice_checksum=None, dev=0):
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    sb, sl, sc = _slice_arrays(checksum_alg, slice_base, slice_len, slice_checksum)
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_decompress_dev(dev, codec, checksum_alg, n, d_src, _ptr(off), _ptr(length), _ptr(sb), _ptr(sl),
                                     _ptr(sc), d_dst, dst_cap, _ptr(dst_off), _ptr(dst_len), C.addressof(total),
                                     _ptr(st), _ptr(bad)), "b2s_decompress_dev")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, status=st[:n], bad_slice=bad[:n])


def decompress_sort_dev(codec, d_src, off, length, d_dst, dst_cap, record_bytes, key_off, key_len,
                        checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None, slice_checksum=None, dev=0):
    """decompress_sort_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_sort_dev", codec, d_src, off, length, d_dst, dst_cap,
                      (record_bytes, key_off, key_len), checksum_alg, (slice_base, slice_len, slice_checksum), dev)


def decompress_sort_rows_dev(codec, d_src, off, length, d_dst, dst_cap, key_type, key_off, key_len, null_field=-1,
                             checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None, slice_checksum=None, dev=0):
    """decompress_sort_rows_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_sort_rows_dev", codec, d_src, off, length, d_dst, dst_cap,
                      (key_type, key_off, key_len, null_field), checksum_alg, (slice_base, slice_len, slice_checksum),
                      dev)


def decompress_aggregate_rows_dev(codec, d_src, off, length, d_dst, dst_cap, key_type, key_off, key_len,
                                  null_field=-1, aggs=(), checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                  slice_checksum=None, dev=0):
    """decompress_aggregate_rows_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_aggregate_rows_dev", codec, d_src, off, length, d_dst, dst_cap,
                      (key_type, key_off, key_len, null_field, *_agg_arrays(aggs)), checksum_alg,
                      (slice_base, slice_len, slice_checksum), dev)


def decompress_sort_rows_keys_dev(codec, d_src, off, length, d_dst, dst_cap, keys, checksum_alg=CHECKSUM_NONE,
                                  slice_base=None, slice_len=None, slice_checksum=None, dev=0):
    """decompress_sort_rows_keys_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_sort_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      _key_arrays(keys), checksum_alg, (slice_base, slice_len, slice_checksum), dev)


def decompress_aggregate_rows_keys_dev(codec, d_src, off, length, d_dst, dst_cap, keys, aggs=(),
                                       checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                       slice_checksum=None, dev=0):
    """decompress_aggregate_rows_keys_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_aggregate_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      (*_key_arrays(keys), *_agg_arrays(aggs)), checksum_alg, (slice_base, slice_len, slice_checksum),
                      dev)


def decompress_join_rows_keys_dev(join_type, codec, d_src, off, length, n_left, d_dst, dst_cap, left_keys, right_keys,
                                  n_left_fields, n_right_fields, left_kinds=None, right_kinds=None,
                                  checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None, slice_checksum=None,
                                  dev=0):
    """decompress_join_rows_keys_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    n, kt, kl, lo, ln, ro, rn, lk, rk = _join_arrays(left_keys, right_keys, left_kinds, right_kinds)
    return _sort_call("b2s_decompress_join_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      (n, kt, kl, lo, ln, ro, rn, n_left_fields, lk, n_right_fields, rk), checksum_alg,
                      (slice_base, slice_len, slice_checksum), dev, lead=(join_type,), before_n=(n_left,))


def decompress_window_rows_keys_dev(codec, d_src, off, length, d_dst, dst_cap, keys, n_partition_keys, n_fields, kinds,
                                    fns, limit=None, checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                    slice_checksum=None, dev=0):
    """decompress_window_rows_keys_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_window_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      _window_arrays(keys, n_partition_keys, n_fields, kinds, fns, limit), checksum_alg,
                      (slice_base, slice_len, slice_checksum), dev)


def decompress_window_frame_rows_keys_dev(codec, d_src, off, length, d_dst, dst_cap, keys, n_partition_keys, n_fields,
                                          kinds, fns, checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                          slice_checksum=None, dev=0):
    """decompress_window_frame_rows_keys_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_window_frame_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      _window_frame_arrays(keys, n_partition_keys, n_fields, kinds, fns), checksum_alg,
                      (slice_base, slice_len, slice_checksum), dev=dev)


def decompress_window_offset_rows_keys_dev(codec, d_src, off, length, d_dst, dst_cap, keys, n_partition_keys, n_fields,
                                           kinds, fns, checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                                           slice_checksum=None, dev=0):
    """decompress_window_offset_rows_keys_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_window_offset_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      _window_offset_arrays(keys, n_partition_keys, n_fields, kinds, fns), checksum_alg,
                      (slice_base, slice_len, slice_checksum), dev=dev)


def decompress_window_aggregate_rows_keys_dev(codec, d_src, off, length, d_dst, dst_cap, keys, n_partition_keys,
                                              n_fields, kinds, fns, checksum_alg=CHECKSUM_NONE, slice_base=None,
                                              slice_len=None, slice_checksum=None, dev=0):
    """decompress_window_aggregate_rows_keys_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    return _sort_call("b2s_decompress_window_aggregate_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      _window_aggregate_arrays(keys, n_partition_keys, n_fields, kinds, fns), checksum_alg,
                      (slice_base, slice_len, slice_checksum), dev)


def partition_compress_dev(codec, d_records, rec_bytes, d_rec_len, d_rec_part, n_records, num_partitions, d_dst,
                           dst_cap, block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """d_*: device addresses (records, u32 lengths, u32 reduce ids, destination arena)"""
    return _partition_call("b2s_partition_compress_dev", codec, level, block_size, checksum_alg, num_partitions,
                           (num_partitions, n_records, d_records, rec_bytes, d_rec_len, d_rec_part), d_dst, dst_cap,
                           dev)


def partition_compress_rows_hash_packed(codec, records, rec_len, keys, num_partitions, dst, block_size=0,
                                        checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_packed of serialized UnsafeRows ([int32 big-endian size][row] each), every record's reduce
    id Spark's pmod(Murmur3Hash(key columns, 42), num_partitions); keys as in decompress_sort_rows_keys_packed, no
    order flags; a type OR-ed with KEY_NULL_SAFE hashes as its (coalesce(v, default), isnull(v)) key pair.
    -> dict(dst_off, dst_len, total, checksums, status)"""
    return _partition_call("b2s_partition_compress_rows_hash_packed", codec, level, block_size, checksum_alg,
                           num_partitions, (num_partitions, *_records(records, rec_len), *_key_arrays(keys)), dst)


def partition_compress_rows_hash_dev(codec, d_records, rec_bytes, d_rec_len, n_records, keys, num_partitions, d_dst,
                                     dst_cap, block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """partition_compress_rows_hash_packed on device addresses (records, u32 lengths, destination arena)"""
    return _partition_call("b2s_partition_compress_rows_hash_dev", codec, level, block_size, checksum_alg,
                           num_partitions,
                           (num_partitions, n_records, d_records, rec_bytes, d_rec_len, *_key_arrays(keys)), d_dst,
                           dst_cap, dev)


def _partial_agg_arrays(aggs):
    """aggs = [(fn, val_type, val_off, val_null_field), ...]: WINDOW_SUM / COUNT / MIN / MAX / AVG / VARIANCE, WINDOW_VAL_* or
    window_val_decimal(p, s) -> (n, fn, val_type, val_off, val_null_field) arrays"""
    aggs = list(aggs)
    cols = list(zip(*aggs)) if aggs else [[0]] * 4
    fn, vt, vo, vn = (np.array(c, dtype=t) for c, t in zip(cols, (np.uint32, np.uint32, np.uint32, np.int32)))
    return len(aggs), fn, vt, vo, vn


def _set_arrays(sets):
    """sets = grouping-set masks -> (n_sets, set_mask array)"""
    sets = list(sets)
    return len(sets), np.ascontiguousarray(sets or [0], dtype=np.uint32)


def aggregate_partition_compress_rows_hash_packed(codec, records, rec_len, keys, aggs, num_partitions, dst,
                                                  block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """Spark's HashAggregateExec(Partial) and its hash exchange: the serialized UnsafeRows grouped by the key columns
    (as in partition_compress_rows_hash_packed), the aggregation buffers of aggs (_partial_agg_arrays) folded per key,
    one partial row per key, hash-partitioned and compressed.  -> dict(dst_off, dst_len, total, checksums, status,
    n_groups)"""
    return _partition_call("b2s_aggregate_partition_compress_rows_hash_packed", codec, level, block_size,
                           checksum_alg, num_partitions,
                           (num_partitions, *_records(records, rec_len), *_key_arrays(keys),
                            *_partial_agg_arrays(aggs)), dst, counts=("n_groups",))


def aggregate_partition_compress_rows_hash_dev(codec, d_records, rec_bytes, d_rec_len, n_records, keys, aggs,
                                               num_partitions, d_dst, dst_cap, block_size=0,
                                               checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """aggregate_partition_compress_rows_hash_packed on device addresses (records, u32 lengths, destination arena)"""
    return _partition_call("b2s_aggregate_partition_compress_rows_hash_dev", codec, level, block_size, checksum_alg,
                           num_partitions,
                           (num_partitions, n_records, d_records, rec_bytes, d_rec_len, *_key_arrays(keys),
                            *_partial_agg_arrays(aggs)), d_dst, dst_cap, dev, counts=("n_groups",))


DISTINCT_ALL_COLUMNS = -1  # B2S_DISTINCT_ALL_COLUMNS: count(DISTINCT every distinct column)


def aggregate_distinct_partition_compress_rows_hash(codec, src, off, length, dst, n_group_keys, keys, aggs, distinct,
                                                    num_partitions, checksum_alg=CHECKSUM_NONE, slice_base=None,
                                                    slice_len=None, slice_checksum=None, block_size=0, level=0,
                                                    dev=None, dst_cap=None):
    """One DISTINCT group's middle stage on a reducer of the exchange by G ++ X: its blocks of the map side's partial
    rows (keys G ++ X, functions aggs) merged per (G, X), folded per G (aggs' buffers merged, distinct's updated over
    their columns), hash-partitioned by G and compressed into dst.  keys = [(key_type, key_len), ...], the first
    n_group_keys G; aggs = [(fn, val_type), ...]; distinct = [(fn, val_type, column or DISTINCT_ALL_COLUMNS), ...].
    dev None: src and dst host arrays; else device addresses (dst_cap required).  -> dict(dst_off, dst_len, total,
    checksums, part_status, counts (input rows, (G, X) groups, rows written), status, bad_slice)"""
    if dev is None:
        src, dst = _as_u8(src), _as_u8(dst)
        dst_cap = dst.size
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    sb, sl, sc = _slice_arrays(checksum_alg, slice_base, slice_len, slice_checksum)
    kt = np.array([k[0] for k in keys] or [0], dtype=np.uint32)
    kl = np.array([k[1] for k in keys] or [0], dtype=np.uint32)
    fn = np.array([a[0] for a in aggs] or [0], dtype=np.uint32)
    vt = np.array([a[1] for a in aggs] or [0], dtype=np.uint32)
    dfn = np.array([a[0] for a in distinct] or [0], dtype=np.uint32)
    dvt = np.array([a[1] for a in distinct] or [0], dtype=np.uint32)
    dcol = np.array([a[2] for a in distinct] or [0], dtype=np.int32)
    dst_off, dst_len, cks, pst = _partition_out(num_partitions)
    total = _u64(0)
    counts = np.zeros(3, dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    symbol = "b2s_decompress_aggregate_distinct_partition_compress_rows_hash_" + ("packed" if dev is None else "dev")
    lead = [] if dev is None else [dev]
    _check(getattr(load(), symbol)(
        *lead, codec, level, block_size, checksum_alg, n, _arg(src), _ptr(off), _ptr(length), _arg(sb), _arg(sl),
        _arg(sc), n_group_keys, len(keys), _ptr(kt), _ptr(kl), len(aggs), _ptr(fn), _ptr(vt), len(distinct), _ptr(dfn),
        _ptr(dvt), _ptr(dcol), num_partitions, _arg(dst), dst_cap, _ptr(dst_off), _ptr(dst_len), C.addressof(total),
        _ptr(cks), _ptr(pst), _ptr(counts), _ptr(st), _ptr(bad)), symbol)
    return dict(dst_off=dst_off, dst_len=dst_len, total=total.value, checksums=cks, part_status=pst,
                counts=[int(c) for c in counts], status=st[:n], bad_slice=bad[:n])


def aggregate_grouping_sets_partition_compress_rows_hash_packed(codec, records, rec_len, keys, aggs, sets,
                                                                num_partitions, dst, block_size=0,
                                                                checksum_alg=CHECKSUM_NONE, level=0):
    """Spark's Expand over grouping sets, then HashAggregateExec(Partial) and its hash exchange: as
    aggregate_partition_compress_rows_hash_packed, each record once per grouping set (sets: one mask per set, bit c for
    key column c), the partial rows keyed by the grouping columns and spark_grouping_id.  -> dict(dst_off, dst_len,
    total, checksums, status, n_groups)"""
    return _partition_call("b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed", codec, level,
                           block_size, checksum_alg, num_partitions,
                           (num_partitions, *_records(records, rec_len), *_key_arrays(keys),
                            *_partial_agg_arrays(aggs), *_set_arrays(sets)), dst, counts=("n_groups",))


def aggregate_grouping_sets_partition_compress_rows_hash_dev(codec, d_records, rec_bytes, d_rec_len, n_records, keys,
                                                             aggs, sets, num_partitions, d_dst, dst_cap, block_size=0,
                                                             checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """aggregate_grouping_sets_partition_compress_rows_hash_packed on device addresses (records, u32 lengths,
    destination arena)"""
    return _partition_call("b2s_aggregate_grouping_sets_partition_compress_rows_hash_dev", codec, level, block_size,
                           checksum_alg, num_partitions,
                           (num_partitions, n_records, d_records, rec_bytes, d_rec_len, *_key_arrays(keys),
                            *_partial_agg_arrays(aggs), *_set_arrays(sets)), d_dst, dst_cap, dev, counts=("n_groups",))


def window_limit_partition_compress_rows_hash_packed(codec, records, rec_len, keys, n_partition_keys, limit_fn, limit,
                                                     num_partitions, dst, block_size=0, checksum_alg=CHECKSUM_NONE,
                                                     level=0):
    """Spark's Sort and WindowGroupLimitExec(Partial), then its exchange: the records sorted by keys (the first
    n_partition_keys the PARTITION BY columns, the rest the ORDER BY columns), those whose limit_fn (WINDOW_ROW_NUMBER,
    WINDOW_RANK or WINDOW_DENSE_RANK) value in their partition is at most limit kept and hash-partitioned by the partition
    columns (none: SinglePartition, num_partitions 1).  -> dict(dst_off, dst_len, total, checksums, status,
    n_out_records)"""
    return _partition_call("b2s_window_limit_partition_compress_rows_hash_packed", codec, level, block_size,
                           checksum_alg, num_partitions,
                           (num_partitions, *_records(records, rec_len), n_partition_keys, *_key_arrays(keys),
                            limit_fn, limit), dst, counts=("n_out_records",))


def window_limit_partition_compress_rows_hash_dev(codec, d_records, rec_bytes, d_rec_len, n_records, keys,
                                                  n_partition_keys, limit_fn, limit, num_partitions, d_dst, dst_cap,
                                                  block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """window_limit_partition_compress_rows_hash_packed on device addresses (records, u32 lengths, destination arena)"""
    return _partition_call("b2s_window_limit_partition_compress_rows_hash_dev", codec, level, block_size, checksum_alg,
                           num_partitions,
                           (num_partitions, n_records, d_records, rec_bytes, d_rec_len, n_partition_keys,
                            *_key_arrays(keys), limit_fn, limit), d_dst, dst_cap, dev, counts=("n_out_records",))


def _bound_arrays(bounds):
    """bounds = the RangePartitioner's bound rows, each framed as UnsafeRowSerializer writes it ([int32 big-endian
    size][row]) -> (n, rows back to back, their lengths)"""
    bounds = [bytes(b) for b in bounds]
    base = np.frombuffer(b"".join(bounds) or b"\0", dtype=np.uint8).copy()
    return len(bounds), base, sum(len(b) for b in bounds), np.array([len(b) for b in bounds] or [0], dtype=np.uint32)


def partition_compress_rows_range_packed(codec, records, rec_len, keys, bounds, dst, block_size=0,
                                         checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_packed of serialized UnsafeRows ([int32 big-endian size][row] each), every record's reduce
    id Spark's RangePartitioner id of its key over the bounds (framed rows, _bound_arrays); len(bounds) + 1 partitions;
    keys as in decompress_sort_rows_keys_packed, order flags included.  -> dict(dst_off, dst_len, total, checksums,
    status)"""
    bounds = _bound_arrays(bounds)
    return _partition_call("b2s_partition_compress_rows_range_packed", codec, level, block_size, checksum_alg,
                           bounds[0] + 1, (*_records(records, rec_len), *_key_arrays(keys), *bounds), dst)


def partition_compress_rows_range_dev(codec, d_records, rec_bytes, d_rec_len, n_records, keys, bounds, d_dst, dst_cap,
                                      block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """partition_compress_rows_range_packed on device addresses (records, u32 lengths, destination arena); the bounds
    stay host memory"""
    bounds = _bound_arrays(bounds)
    return _partition_call("b2s_partition_compress_rows_range_dev", codec, level, block_size, checksum_alg,
                           bounds[0] + 1,
                           (n_records, d_records, rec_bytes, d_rec_len, *_key_arrays(keys), *bounds), d_dst,
                           dst_cap, dev)


def partition_compress_rows_round_robin_packed(codec, records, rec_len, num_partitions, start_position, sort_rows,
                                               dst, block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_packed of serialized UnsafeRows ([int32 big-endian size][row] each) in Spark's repartition(n)
    order and ids: sorted by (row hash, row bytes) when sort_rows and num_partitions > 1, then the k-th row to
    (start_position + 1 + k) % num_partitions.  -> dict(dst_off, dst_len, total, checksums, status)"""
    return _partition_call("b2s_partition_compress_rows_round_robin_packed", codec, level, block_size, checksum_alg,
                           num_partitions,
                           (num_partitions, start_position, sort_rows, *_records(records, rec_len)), dst)


def partition_compress_rows_round_robin_dev(codec, d_records, rec_bytes, d_rec_len, n_records, num_partitions,
                                            start_position, sort_rows, d_dst, dst_cap, block_size=0,
                                            checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """partition_compress_rows_round_robin_packed on device addresses (records, u32 lengths, destination arena)"""
    return _partition_call("b2s_partition_compress_rows_round_robin_dev", codec, level, block_size, checksum_alg,
                           num_partitions,
                           (num_partitions, start_position, sort_rows, n_records, d_records, rec_bytes, d_rec_len),
                           d_dst, dst_cap, dev)


# ---------------------------------------------------------------------------------------------------------------
# exchange cache: map outputs kept resident in HBM for reducers on the same device
# ---------------------------------------------------------------------------------------------------------------
def exchange_set_budget(nbytes, dev=0):
    """per-device budget in bytes of cached records and of the row entries' record boundaries (8 per record); 0 (the
    default) turns the cache off"""
    _check(load().b2s_exchange_set_budget(dev, nbytes), "b2s_exchange_set_budget")


def partition_compress_cached_packed(shuffle_id, map_id, codec, records, rec_len, rec_part, num_partitions, dst,
                                     block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_packed that also keeps the partitioned records as the cache entry (shuffle_id, map_id).
    -> dict(dst_off, dst_len, total, checksums, status, cached)"""
    return _partition_call("b2s_partition_compress_cached_packed", codec, level, block_size, checksum_alg,
                           num_partitions,
                           (num_partitions, *_records(records, rec_len), np.ascontiguousarray(rec_part, np.uint32)),
                           dst, lead=(shuffle_id, map_id), counts=("cached",))


def exchange_lookup(shuffle_id, start_reduce, end_reduce, map_ids):
    """-> (hits, lengths): lengths[i] = bytes of the range of map_ids[i], NOT_RESIDENT when it is not resident"""
    ids = np.ascontiguousarray(map_ids, dtype=np.int64)
    ln = np.zeros(max(ids.size, 1), dtype=np.uint64)
    rc = load().b2s_exchange_lookup(shuffle_id, start_reduce, end_reduce, ids.size, _ptr(ids), _ptr(ln))
    if rc < 0:
        raise B2SError(rc, "b2s_exchange_lookup")
    return rc, ln[: ids.size]


def exchange_read_packed(shuffle_id, start_reduce, end_reduce, map_ids, dst):
    """the cached ranges back to back into dst.  -> dict(dst_off, dst_len, total, status)"""
    ids = np.ascontiguousarray(map_ids, dtype=np.int64)
    dst = _as_u8(dst)
    n = ids.size
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_exchange_read_packed(shuffle_id, start_reduce, end_reduce, n, _ptr(ids), _ptr(dst), dst.size,
                                           _ptr(dst_off), _ptr(dst_len), C.addressof(total), _ptr(st)),
           "b2s_exchange_read_packed")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, status=st[:n])


def _exchange_sources(map_ids, cached):
    return (np.ascontiguousarray(map_ids, dtype=np.int64),
            np.ascontiguousarray(np.asarray(cached, dtype=bool), dtype=np.uint8))


def exchange_read_sort_packed(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, src, off, length, dst,
                              record_bytes, key_off, key_len, checksum_alg=CHECKSUM_NONE, slice_base=None,
                              slice_len=None, slice_checksum=None):
    """decompress_sort_packed over sources of which those with cached[i] set are the cached range of map_ids[i].
    -> dict(total, n_records, status, bad_slice)"""
    ids, cm = _exchange_sources(map_ids, cached)
    return _sort_call("b2s_exchange_read_sort_packed", codec, src, off, length, dst, None,
                      (record_bytes, key_off, key_len), checksum_alg, (slice_base, slice_len, slice_checksum),
                      lead=(shuffle_id, start_reduce, end_reduce, ids, cm), n=ids.size)


def exchange_read_sort_dev(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, d_src, off, length, d_dst,
                           dst_cap, record_bytes, key_off, key_len, checksum_alg=CHECKSUM_NONE, slice_base=None,
                           slice_len=None, slice_checksum=None, dev=0):
    """exchange_read_sort_packed with the fetched blocks (d_src) and the output (d_dst) in device memory"""
    ids, cm = _exchange_sources(map_ids, cached)
    return _sort_call("b2s_exchange_read_sort_dev", codec, d_src, off, length, d_dst, dst_cap,
                      (record_bytes, key_off, key_len), checksum_alg, (slice_base, slice_len, slice_checksum), dev,
                      lead=(shuffle_id, start_reduce, end_reduce, ids, cm), n=ids.size)


def partition_compress_rows_hash_cached_packed(shuffle_id, map_id, codec, records, rec_len, keys, num_partitions, dst,
                                               block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_rows_hash_packed that also keeps the partitioned rows and their record boundaries as the cache
    entry (shuffle_id, map_id).  -> dict(dst_off, dst_len, total, checksums, status, cached)"""
    return _partition_call("b2s_partition_compress_rows_hash_cached_packed", codec, level, block_size, checksum_alg,
                           num_partitions, (num_partitions, *_records(records, rec_len), *_key_arrays(keys)), dst,
                           lead=(shuffle_id, map_id), counts=("cached",))


def partition_compress_rows_range_cached_packed(shuffle_id, map_id, codec, records, rec_len, keys, bounds, dst,
                                                block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_rows_range_packed that also keeps the partitioned rows and their record boundaries as the
    cache entry (shuffle_id, map_id).  -> dict(dst_off, dst_len, total, checksums, status, cached)"""
    bounds = _bound_arrays(bounds)
    return _partition_call("b2s_partition_compress_rows_range_cached_packed", codec, level, block_size, checksum_alg,
                           bounds[0] + 1, (*_records(records, rec_len), *_key_arrays(keys), *bounds), dst,
                           lead=(shuffle_id, map_id), counts=("cached",))


def partition_compress_rows_round_robin_cached_packed(shuffle_id, map_id, codec, records, rec_len, num_partitions,
                                                      start_position, sort_rows, dst, block_size=0,
                                                      checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_rows_round_robin_packed that also keeps the partitioned rows and their record boundaries as
    the cache entry (shuffle_id, map_id).  -> dict(dst_off, dst_len, total, checksums, status, cached)"""
    return _partition_call("b2s_partition_compress_rows_round_robin_cached_packed", codec, level, block_size,
                           checksum_alg, num_partitions,
                           (num_partitions, start_position, sort_rows, *_records(records, rec_len)), dst,
                           lead=(shuffle_id, map_id), counts=("cached",))


def exchange_read_sort_rows_keys_packed(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, src, off,
                                        length, dst, keys, checksum_alg=CHECKSUM_NONE, slice_base=None,
                                        slice_len=None, slice_checksum=None):
    """decompress_sort_rows_keys_packed over sources of which those with cached[i] set are the cached range of
    map_ids[i].  -> dict(total, n_records, status, bad_slice)"""
    ids, cm = _exchange_sources(map_ids, cached)
    return _sort_call("b2s_exchange_read_sort_rows_keys_packed", codec, src, off, length, dst, None, _key_arrays(keys),
                      checksum_alg, (slice_base, slice_len, slice_checksum),
                      lead=(shuffle_id, start_reduce, end_reduce, ids, cm), n=ids.size)


def exchange_read_sort_rows_keys_dev(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, d_src, off, length,
                                     d_dst, dst_cap, keys, checksum_alg=CHECKSUM_NONE, slice_base=None,
                                     slice_len=None, slice_checksum=None, dev=0):
    """exchange_read_sort_rows_keys_packed with the fetched blocks (d_src) and the output (d_dst) in device memory"""
    ids, cm = _exchange_sources(map_ids, cached)
    return _sort_call("b2s_exchange_read_sort_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      _key_arrays(keys), checksum_alg, (slice_base, slice_len, slice_checksum), dev,
                      lead=(shuffle_id, start_reduce, end_reduce, ids, cm), n=ids.size)


def exchange_read_aggregate_rows_keys_packed(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, src, off,
                                             length, dst, keys, aggs=(), checksum_alg=CHECKSUM_NONE, slice_base=None,
                                             slice_len=None, slice_checksum=None):
    """decompress_aggregate_rows_keys_packed over sources of which those with cached[i] set are the cached range of
    map_ids[i].  -> dict(total, n_records, n_groups, status, bad_slice)"""
    ids, cm = _exchange_sources(map_ids, cached)
    return _sort_call("b2s_exchange_read_aggregate_rows_keys_packed", codec, src, off, length, dst, None,
                      (*_key_arrays(keys), *_agg_arrays(aggs)), checksum_alg, (slice_base, slice_len, slice_checksum),
                      lead=(shuffle_id, start_reduce, end_reduce, ids, cm), n=ids.size)


def exchange_read_aggregate_rows_keys_dev(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, d_src, off,
                                          length, d_dst, dst_cap, keys, aggs=(), checksum_alg=CHECKSUM_NONE,
                                          slice_base=None, slice_len=None, slice_checksum=None, dev=0):
    """exchange_read_aggregate_rows_keys_packed with the fetched blocks (d_src) and the output (d_dst) in device
    memory"""
    ids, cm = _exchange_sources(map_ids, cached)
    return _sort_call("b2s_exchange_read_aggregate_rows_keys_dev", codec, d_src, off, length, d_dst, dst_cap,
                      (*_key_arrays(keys), *_agg_arrays(aggs)), checksum_alg, (slice_base, slice_len, slice_checksum),
                      dev, lead=(shuffle_id, start_reduce, end_reduce, ids, cm), n=ids.size)


def exchange_remove(shuffle_id, map_id=-1):
    """removes (shuffle_id, map_id), or every map output of the shuffle (map_id -1), on every device -> count"""
    rc = load().b2s_exchange_remove(shuffle_id, map_id)
    if rc < 0:
        raise B2SError(rc, "b2s_exchange_remove")
    return rc
