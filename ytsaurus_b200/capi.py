"""ctypes binding of include/ytgpu.h (the C-ABI shared library libytgpu.so).

There is no CPU fallback: importing works anywhere (so the symbol table can be
checked on a CPU box), but creating a context without a CUDA device raises.
"""
from __future__ import annotations

import ctypes as C
import os
import struct

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libytgpu.so")

MEM_DEVICE, MEM_HOST = 0, 1

OK = 0
ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, ERR_CUDA, ERR_OUT_OF_MEMORY, ERR_SCHEMA_VIOLATION = 1, 2, 3, 4, 5
ERR_PARTITION_BAD_TYPE, ERR_PARTITION_NEGATIVE, ERR_PARTITION_OUT_OF_BOUNDS, ERR_PARTITION_NO_COLUMN = 10, 11, 12, 13

PARTITION_ORDERED, PARTITION_HASH, PARTITION_COLUMN = 0, 1, 2
TYPE_NULL, TYPE_INT64, TYPE_UINT64, TYPE_DOUBLE, TYPE_BOOLEAN, TYPE_STRING = 0x02, 0x03, 0x04, 0x05, 0x06, 0x10
CMP_NONE, CMP_LT, CMP_LE, CMP_GT, CMP_GE, CMP_EQ, CMP_NE = range(7)

KC_RADIX_PASS, KC_GATHER, KC_EXTRACT, KC_HISTOGRAM, KC_PARTITION, KC_GROUPBY, KC_DECODE, KC_PASS_SKIPPED, KC_SCATTER, \
    KC_SHUFFLE_SYNC, KC_REDUCE, KC_JOIN = range(12)
MAX_SHUFFLE_RANKS = 32


class Error(C.Structure):
    _fields_ = [("code", C.c_int32), ("cuda_error", C.c_int32), ("message", C.c_char * 248)]


class RowsetView(C.Structure):
    _fields_ = [("values", C.c_void_p), ("row_count", C.c_uint64), ("value_count", C.c_uint32),
                ("reserved", C.c_uint32), ("string_heap", C.c_void_p), ("string_heap_bytes", C.c_uint64),
                ("mem", C.c_int32)]


class FixedRowsView(C.Structure):
    _fields_ = [("rows", C.c_void_p), ("row_count", C.c_uint64), ("row_bytes", C.c_uint32), ("mem", C.c_int32)]


class KeyColumn(C.Structure):
    _fields_ = [("index", C.c_uint32), ("width", C.c_uint32), ("type", C.c_uint8), ("descending", C.c_uint8),
                ("required", C.c_uint8), ("reserved", C.c_uint8)]


class SortSpec(C.Structure):
    _fields_ = [("columns", C.POINTER(KeyColumn)), ("column_count", C.c_uint32)]


class PartitionSpec(C.Structure):
    _fields_ = [("kind", C.c_int32), ("partition_count", C.c_int32), ("key", SortSpec),
                ("bounds", C.c_void_p), ("bounds_heap", C.c_void_p), ("bounds_heap_bytes", C.c_uint64),
                ("bound_value_count", C.c_uint32), ("bound_prefix_length", C.c_void_p),
                ("bound_inclusive", C.c_void_p), ("key_column_count", C.c_int32), ("salt", C.c_uint64),
                ("partition_column_id", C.c_uint16)]


class ColumnView(C.Structure):
    _fields_ = [("start_index", C.c_int64), ("value_count", C.c_int64), ("value_type", C.c_uint8),
                ("has_values", C.c_uint8), ("zigzag", C.c_uint8), ("bit_width", C.c_uint8),
                ("reserved", C.c_uint32), ("base_value", C.c_uint64), ("values", C.c_void_p),
                ("values_count", C.c_uint64), ("null_bitmap", C.c_void_p), ("dictionary_indexes", C.c_void_p),
                ("dictionary_index_count", C.c_uint64), ("rle_indexes", C.c_void_p), ("rle_count", C.c_uint64),
                ("mem", C.c_int32)]


class ShuffleStats(C.Structure):
    _fields_ = [("rows_in", C.c_uint64), ("rows_out", C.c_uint64), ("sent", C.c_uint64 * 32), ("received", C.c_uint64 * 32),
                ("world", C.c_uint32), ("maniac", C.c_uint32)]


class Predicate(C.Structure):
    _fields_ = [("op", C.c_int32), ("reserved", C.c_int32), ("constant", C.c_uint64)]


class GroupByResult(C.Structure):
    _fields_ = [("group_count", C.c_uint64), ("keys", C.c_void_p), ("key_null", C.c_void_p),
                ("sums", C.c_void_p), ("sum_null", C.c_void_p), ("counts", C.c_void_p), ("capacity", C.c_uint64),
                ("first_rows", C.c_void_p), ("mins", C.c_void_p), ("maxs", C.c_void_p)]


# ytgpu_integer_segment (80 bytes), as a numpy record
INTEGER_SEGMENT_DTYPE = np.dtype([
    ("type", "<u4"), ("row_count", "<u4"), ("chunk_row_count", "<u8"), ("min_value", "<u8"), ("data_offset", "<u8"),
    ("data_bytes", "<u8"), ("part_bytes", "<u8", (3,)), ("values_size", "<u4"), ("ids_size", "<u4"),
    ("row_indexes_size", "<u4"), ("values_width", "u1"), ("ids_width", "u1"), ("row_indexes_width", "u1"), ("direct", "u1"),
])
assert INTEGER_SEGMENT_DTYPE.itemsize == 80

PLAIN_SEGMENT_DTYPE = np.dtype([("row_count", "<u4"), ("reserved", "<u4"), ("chunk_row_count", "<u8"), ("data_offset", "<u8"),
                                ("data_bytes", "<u8"), ("part_bytes", "<u8", (3,))])
assert PLAIN_SEGMENT_DTYPE.itemsize == 56

STRING_SEGMENT_DTYPE = np.dtype([
    ("type", "<u4"), ("row_count", "<u4"), ("chunk_row_count", "<u8"), ("data_offset", "<u8"), ("data_bytes", "<u8"),
    ("part_bytes", "<u8", (4,)), ("expected_length", "<u4"), ("offsets_size", "<u4"), ("ids_size", "<u4"),
    ("row_indexes_size", "<u4"), ("offsets_width", "u1"), ("ids_width", "u1"), ("row_indexes_width", "u1"), ("direct", "u1"),
    ("reserved", "<u4")])
assert STRING_SEGMENT_DTYPE.itemsize == 88

# Every symbol include/ytgpu.h declares (tests check that the library exports all of them).
EXPORTED_SYMBOLS = [
    "ytgpu_abi_version", "ytgpu_context_create", "ytgpu_context_destroy", "ytgpu_context_synchronize",
    "ytgpu_context_launch_count", "ytgpu_context_kernel_ms", "ytgpu_context_reset_timers",
    "ytgpu_context_enable_timers", "ytgpu_context_last_sort_passes", "ytgpu_host_alloc", "ytgpu_host_free",
    "ytgpu_sort_rowset", "ytgpu_sort_fixed_rows", "ytgpu_merge_sorted_runs", "ytgpu_join_sorted_runs",
    "ytgpu_partition_rowset", "ytgpu_partition_rowset_slabs", "ytgpu_partition_fixed_rows", "ytgpu_farm_fingerprint_rowset",
    "ytgpu_peer_buffer_create", "ytgpu_peer_buffer_destroy", "ytgpu_peer_buffer_open", "ytgpu_peer_buffer_close",
    "ytgpu_scatter_rows_to_peers", "ytgpu_shuffle_create", "ytgpu_shuffle_connect", "ytgpu_shuffle_sort",
    "ytgpu_shuffle_destroy", "ytgpu_reduce_sorted_fixed_rows", "ytgpu_context_set_option", "ytgpu_context_notify", "ytgpu_decode_horizontal_block", "ytgpu_encode_horizontal_block",
    "ytgpu_decode_column", "ytgpu_decode_string_offsets", "ytgpu_decode_string_pointers_and_lengths", "ytgpu_scan_filter_groupby", "ytgpu_scan_filter_groupby_multi",
    "ytgpu_scan_filter_groupby_multi_strings", "ytgpu_evaluate_filter", "ytgpu_evaluate_expression",
    "ytgpu_evaluate_expression_strings",
    "ytgpu_convert_integer_column", "ytgpu_encode_integer_column", "ytgpu_encode_double_column", "ytgpu_encode_boolean_column", "ytgpu_encode_string_column", "ytgpu_decode_string_segment", "ytgpu_string_value_ids", "ytgpu_extract_column",
    "ytgpu_block_agg_state_init", "ytgpu_block_combine_all",
    "ytgpu_build_bitmap_from_flags", "ytgpu_build_bytemap_from_flags", "ytgpu_count_flags", "ytgpu_build_dictionary_indexes",
    "ytgpu_count_total_string_length", "ytgpu_translate_rle_indexes", "ytgpu_context_get_option", "ytgpu_convert_ch_column_to_values", "ytgpu_convert_string_column_to_ch", "ytgpu_decode_column_typed",
    "ytgpu_hash_join", "ytgpu_gather_column", "ytgpu_gather_string_column", "ytgpu_order_rows",
    "ytgpu_join_table_build", "ytgpu_join_table_probe", "ytgpu_join_table_destroy",
    "ytgpu_join_table_build_strings", "ytgpu_join_table_probe_strings",
    "ytgpu_groupby_table_create", "ytgpu_groupby_table_update", "ytgpu_groupby_table_result", "ytgpu_groupby_table_destroy",
    "ytgpu_groupby_table_create_strings", "ytgpu_groupby_table_update_strings", "ytgpu_groupby_table_result_strings",
]

FLAGS_DICTIONARY_ZERO, FLAGS_BITMAP = 0, 1


(CH_INT8, CH_INT16, CH_INT32, CH_INT64, CH_UINT8, CH_UINT16, CH_UINT32, CH_UINT64, CH_FLOAT32, CH_FLOAT64, CH_BOOL, CH_STRING,
 CH_DATE, CH_DATE32, CH_DATETIME, CH_DATETIME64, CH_TIMESTAMP) = range(1, 18)


class ChColumn(C.Structure):
    _fields_ = [("type", C.c_int32), ("mem", C.c_int32), ("data", C.c_void_p), ("offsets", C.c_void_p), ("chars_bytes", C.c_uint64),
                ("null_map", C.c_void_p), ("time_adjustment", C.c_int64), ("row_count", C.c_uint64)]


class StringColumnView(C.Structure):
    _fields_ = [("offsets", C.c_void_p), ("string_count", C.c_uint64), ("avg_length", C.c_uint32), ("mem", C.c_int32),
                ("chars", C.c_void_p), ("chars_bytes", C.c_uint64), ("dictionary_indexes", C.c_void_p),
                ("dictionary_index_count", C.c_uint64), ("rle_indexes", C.c_void_p), ("rle_count", C.c_uint64),
                ("start_index", C.c_int64), ("value_count", C.c_int64)]


class FlagSource(C.Structure):
    _fields_ = [("kind", C.c_int32), ("reserved", C.c_int32), ("data", C.c_void_p), ("data_count", C.c_uint64),
                ("rle_indexes", C.c_void_p), ("rle_count", C.c_uint64)]


AGG_SUM, AGG_MIN, AGG_MAX, AGG_COUNT, AGG_AVG, AGG_ARGMIN, AGG_ARGMAX, AGG_FIRST = range(8)
JOIN_INNER, JOIN_LEFT, JOIN_SEMI, JOIN_ANTI = 0, 1, 2, 3
JOIN_NULLS_EQUAL, JOIN_NULLS_NEVER_MATCH = 0, 1
JOIN_NO_ROW = 0xFFFFFFFF
JOIN_MAX_KEYS = 8


class Aggregate(C.Structure):
    _fields_ = [("op", C.c_int32), ("column", C.c_int32), ("by_column", C.c_int32), ("reserved", C.c_int32)]


class StringColumn(C.Structure):
    _fields_ = [("heap", C.c_void_p), ("heap_bytes", C.c_uint64), ("starts", C.c_void_p), ("lengths", C.c_void_p),
                ("null_bytemap", C.c_void_p), ("row_count", C.c_uint64), ("mem", C.c_int32), ("reserved", C.c_int32)]


ORDER_MAX_ITEMS = 32
ORDER_MAX_ROWS = 1 << 30  # exclusive


class OrderItem(C.Structure):
    _fields_ = [("column", C.c_uint32), ("is_string", C.c_uint8), ("descending", C.c_uint8), ("reserved", C.c_uint16)]


(FILTER_COMPARE, FILTER_COMPARE_COLUMNS, FILTER_IN, FILTER_STARTS_WITH, FILTER_IS_NULL, FILTER_IS_NOT_NULL, FILTER_AND, FILTER_OR,
 FILTER_NOT, FILTER_CONTAINS, FILTER_LIKE) = range(1, 12)
FILTER_MAX_NODES, FILTER_MAX_DEPTH, FILTER_MAX_IN_ENTRIES, FILTER_MAX_STRING_CONSTANT_BYTES = 64, 16, 65536, 1 << 20
FILTER_MAX_PATTERN_POSITIONS, FILTER_MAX_PATTERN_BYTES = 256, 32768


class FilterNode(C.Structure):
    _fields_ = [("op", C.c_int32), ("cmp", C.c_int32), ("column", C.c_int32), ("column2", C.c_int32), ("constant", C.c_uint64),
                ("length", C.c_uint32), ("reserved", C.c_uint32)]


(EXPR_COLUMN, EXPR_CONSTANT, EXPR_ADD, EXPR_SUB, EXPR_MUL, EXPR_DIV, EXPR_MOD, EXPR_NEG, EXPR_BIT_AND, EXPR_BIT_OR, EXPR_BIT_XOR,
 EXPR_BIT_NOT, EXPR_CAST, EXPR_IF_NULL, EXPR_CONCAT, EXPR_LOWER, EXPR_UPPER, EXPR_FARM_HASH) = range(1, 19)
(EXPR_COMPARE, EXPR_AND, EXPR_OR, EXPR_NOT, EXPR_IS_NULL, EXPR_IS_NOT_NULL, EXPR_IF) = range(19, 26)
EXPR_IN, EXPR_STARTS_WITH, EXPR_CONTAINS, EXPR_LIKE = range(26, 30)
EXPR_TIMESTAMP_FLOOR, EXPR_FORMAT_TIMESTAMP = 30, 31  # FORMAT_TIMESTAMP: ytgpu_evaluate_expression_strings only
TIMESTAMP_HOUR, TIMESTAMP_DAY, TIMESTAMP_WEEK, TIMESTAMP_MONTH, TIMESTAMP_YEAR = range(5)  # TIMESTAMP_FLOOR's `column`
# ytgpu_evaluate_expression_strings only
EXPR_STRING_OPS = (EXPR_CONCAT, EXPR_LOWER, EXPR_UPPER, EXPR_FARM_HASH)
EXPR_PREDICATE_OPS = (EXPR_IN, EXPR_STARTS_WITH, EXPR_CONTAINS, EXPR_LIKE)
EXPR_MAX_NODES, EXPR_MAX_DEPTH = 64, 16
EXPR_MAX_PIECES, EXPR_MAX_HASH_OPERANDS, EXPR_MAX_STRING_CONSTANT_BYTES = 16, 16, 1 << 20
EXPR_MAX_FORMATTED_BYTES = 64


class ExprNode(C.Structure):
    _fields_ = [("op", C.c_int32), ("column", C.c_int32), ("type", C.c_uint8), ("reserved", C.c_uint8 * 7), ("constant", C.c_uint64)]


class ExprConstants:
    """The string_constants of ytgpu_evaluate_expression_strings, built node by node: each method appends what a node
    names and returns that node's `constant`.  bytes(self) is the buffer to pass."""

    def __init__(self):
        self.data = bytearray()

    def __bytes__(self):
        return bytes(self.data)

    def string(self, s: bytes) -> int:
        """A STRING CONSTANT, or the prefix / needle / pattern of STARTS_WITH, CONTAINS and LIKE."""
        off = len(self.data)
        self.data += s
        return (off << 32) | len(s)

    def in_list(self, values) -> int:
        """An IN list: bytes entries for a STRING operand; otherwise numbers, an int being its bit pattern (taken mod
        2^64, so -1 is INT64 -1) and a float a DOUBLE's.  The entries go at an 8-byte boundary, the strings before them."""
        entries = []
        for v in values:
            if isinstance(v, (bytes, bytearray)):
                entries.append(self.string(bytes(v)))
            elif isinstance(v, float):
                entries.append(struct.unpack("<Q", struct.pack("<d", v))[0])
            else:
                entries.append(int(v) & 0xFFFFFFFFFFFFFFFF)
        self.data += bytes(-len(self.data) % 8)
        off = len(self.data)
        self.data += struct.pack(f"<{len(entries)}Q", *entries)
        return (off << 32) | len(entries)


class GroupByMultiResult(C.Structure):
    _fields_ = [("group_count", C.c_uint64), ("capacity", C.c_uint64), ("keys", C.POINTER(C.c_void_p)),
                ("key_null", C.POINTER(C.c_void_p)), ("values", C.POINTER(C.c_void_p)), ("value_null", C.POINTER(C.c_void_p)),
                ("counts", C.c_void_p), ("first_rows", C.c_void_p)]


class GroupByStringKeys(C.Structure):
    _fields_ = [("heap", C.c_void_p), ("heap_capacity", C.c_uint64), ("heap_bytes", C.c_uint64), ("starts", C.c_void_p),
                ("lengths", C.c_void_p), ("null_bytemap", C.c_void_p)]


class ArrowArray(C.Structure):
    _fields_ = [("values", C.c_void_p), ("validity", C.c_void_p), ("offset", C.c_int64), ("length", C.c_int64),
                ("value_type", C.c_uint8), ("nullable", C.c_uint8), ("reserved", C.c_uint16), ("mem", C.c_int32)]


class BlockAggState(C.Structure):
    _fields_ = [("sum", C.c_uint64), ("min_value", C.c_uint64), ("max_value", C.c_uint64), ("count", C.c_uint64),
                ("count_all", C.c_uint64), ("sum_valid", C.c_uint8), ("min_valid", C.c_uint8), ("max_valid", C.c_uint8),
                ("value_type", C.c_uint8), ("reserved", C.c_uint32)]


class YtGpuError(RuntimeError):
    def __init__(self, code: int, message: str, cuda_error: int = 0):
        super().__init__(f"ytgpu error {code}: {message}")
        self.code = code
        self.cuda_error = cuda_error
        self.message = message


_lib = None


def load() -> C.CDLL:
    """Loads libytgpu.so; fails loudly when the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the ytgpu hot path)")
    lib = C.CDLL(LIB_PATH)
    lib.ytgpu_abi_version.restype = C.c_int
    lib.ytgpu_context_create.argtypes = [C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(Error)]
    lib.ytgpu_context_destroy.argtypes = [C.c_void_p]
    lib.ytgpu_context_destroy.restype = None
    lib.ytgpu_context_synchronize.argtypes = [C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_context_launch_count.argtypes = [C.c_void_p]
    lib.ytgpu_context_launch_count.restype = C.c_uint64
    lib.ytgpu_context_kernel_ms.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]
    lib.ytgpu_context_kernel_ms.restype = C.c_double
    lib.ytgpu_context_reset_timers.argtypes = [C.c_void_p]
    lib.ytgpu_context_reset_timers.restype = None
    lib.ytgpu_context_enable_timers.argtypes = [C.c_void_p, C.c_int]
    lib.ytgpu_context_enable_timers.restype = None
    lib.ytgpu_context_last_sort_passes.argtypes = [C.c_void_p]
    lib.ytgpu_context_last_sort_passes.restype = C.c_uint64
    lib.ytgpu_host_alloc.argtypes = [C.c_size_t]
    lib.ytgpu_host_alloc.restype = C.c_void_p
    lib.ytgpu_host_free.argtypes = [C.c_void_p]
    lib.ytgpu_host_free.restype = None
    lib.ytgpu_sort_rowset.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.POINTER(SortSpec), C.c_void_p,
                                      C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_sort_fixed_rows.argtypes = [C.c_void_p, C.POINTER(FixedRowsView), C.POINTER(SortSpec), C.c_void_p,
                                          C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_merge_sorted_runs.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.POINTER(SortSpec), C.c_void_p,
                                            C.c_uint32, C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_join_sorted_runs.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.POINTER(SortSpec), C.c_uint32, C.c_void_p,
                                           C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_scan_filter_groupby_multi.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                                    C.c_void_p, C.c_int32, C.c_uint64, C.POINTER(GroupByMultiResult), C.c_int,
                                                    C.POINTER(Error)]
    lib.ytgpu_scan_filter_groupby_multi_strings.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                                            C.c_uint32, C.c_void_p, C.c_int32, C.c_uint64, C.POINTER(GroupByMultiResult),
                                                            C.c_int, C.c_void_p, C.c_uint32, C.POINTER(Error)]
    lib.ytgpu_evaluate_filter.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                          C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                          C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_evaluate_expression.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_evaluate_expression_strings.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                                      C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                                      C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8),
                                                      C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_partition_rowset.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.POINTER(PartitionSpec), C.c_void_p,
                                           C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_partition_rowset_slabs.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.POINTER(PartitionSpec), C.c_void_p, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_partition_fixed_rows.argtypes = [C.c_void_p, C.POINTER(FixedRowsView), C.POINTER(PartitionSpec),
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_peer_buffer_create.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_peer_buffer_destroy.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_peer_buffer_open.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(Error)]
    lib.ytgpu_peer_buffer_close.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_scatter_rows_to_peers.argtypes = [C.c_void_p, C.POINTER(FixedRowsView), C.c_void_p, C.c_int32, C.c_void_p,
                                                C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_shuffle_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(C.c_void_p), C.c_void_p,
                                         C.POINTER(Error)]
    lib.ytgpu_shuffle_connect.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_shuffle_sort.argtypes = [C.c_void_p, C.POINTER(FixedRowsView), C.POINTER(SortSpec), C.c_void_p, C.c_uint64,
                                       C.POINTER(C.c_uint64), C.POINTER(ShuffleStats), C.POINTER(Error)]
    lib.ytgpu_shuffle_destroy.argtypes = [C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_reduce_sorted_fixed_rows.argtypes = [C.c_void_p, C.POINTER(FixedRowsView), C.c_uint32, C.c_uint32, C.c_uint8, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(Error)]
    lib.ytgpu_context_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.POINTER(Error)]
    lib.ytgpu_convert_ch_column_to_values.argtypes = [C.c_void_p, C.POINTER(ChColumn), C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_convert_string_column_to_ch.argtypes = [C.c_void_p, C.POINTER(StringColumnView), C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                                      C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_context_get_option.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(Error)]
    lib.ytgpu_context_notify.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_decode_horizontal_block.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
                                                  C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_encode_horizontal_block.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.c_void_p, C.c_void_p, C.c_uint64,
                                                  C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_farm_fingerprint_rowset.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.c_uint32, C.c_void_p,
                                                  C.c_int, C.POINTER(Error)]
    lib.ytgpu_decode_column.argtypes = [C.c_void_p, C.POINTER(ColumnView), C.c_void_p, C.c_void_p, C.c_int,
                                        C.POINTER(Error)]
    lib.ytgpu_decode_column_typed.argtypes = [C.c_void_p, C.POINTER(ColumnView), C.c_uint32, C.c_void_p, C.c_void_p, C.c_int,
                                              C.POINTER(Error)]
    lib.ytgpu_decode_string_offsets.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64, C.c_int64,
                                                C.c_void_p, C.c_int, C.POINTER(Error)]
    for fn in (lib.ytgpu_build_bitmap_from_flags, lib.ytgpu_build_bytemap_from_flags):
        fn.argtypes = [C.c_void_p, C.POINTER(FlagSource), C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_count_flags.argtypes = [C.c_void_p, C.POINTER(FlagSource), C.c_int64, C.c_int64, C.POINTER(C.c_int64), C.c_int,
                                      C.POINTER(Error)]
    lib.ytgpu_build_dictionary_indexes.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int64, C.c_int64,
                                                   C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_count_total_string_length.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int64,
                                                    C.c_int64, C.POINTER(C.c_int64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_translate_rle_indexes.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p,
                                                C.c_int, C.POINTER(Error)]
    lib.ytgpu_decode_string_pointers_and_lengths.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p,
                                                             C.c_int, C.POINTER(Error)]
    lib.ytgpu_scan_filter_groupby.argtypes = [C.c_void_p, C.POINTER(ColumnView), C.POINTER(ColumnView),
                                              C.POINTER(Predicate), C.c_uint64, C.POINTER(GroupByResult), C.c_int,
                                              C.POINTER(Error)]
    lib.ytgpu_convert_integer_column.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.c_uint32, C.c_uint8, C.c_void_p,
                                                 C.c_void_p, C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_encode_integer_column.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_uint32,
                                                C.c_uint64, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                                C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(Error)]
    for fn in (lib.ytgpu_encode_double_column, lib.ytgpu_encode_boolean_column):
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64,
                       C.POINTER(C.c_uint64), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(Error)]
    lib.ytgpu_encode_string_column.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                               C.c_uint32, C.c_uint64, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64,
                                               C.POINTER(C.c_uint64), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(Error)]
    lib.ytgpu_decode_string_segment.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                C.POINTER(Error)]
    lib.ytgpu_string_value_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                           C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_hash_join.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64,
                                    C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_join_table_build.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.POINTER(C.c_void_p), C.POINTER(Error)]
    lib.ytgpu_join_table_probe.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64,
                                           C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_join_table_destroy.argtypes = [C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_join_table_build_strings.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int,
                                                   C.POINTER(C.c_void_p), C.POINTER(Error)]
    lib.ytgpu_join_table_probe_strings.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int,
                                                   C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_groupby_table_create.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                               C.c_uint32, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(Error)]
    lib.ytgpu_groupby_table_update.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                               C.c_uint32, C.c_void_p, C.c_int32, C.POINTER(Error)]
    lib.ytgpu_groupby_table_result.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(GroupByMultiResult), C.c_void_p, C.c_uint32, C.c_int,
                                               C.POINTER(Error)]
    lib.ytgpu_groupby_table_destroy.argtypes = [C.c_void_p, C.POINTER(Error)]
    lib.ytgpu_groupby_table_create_strings.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32,
                                                       C.c_void_p, C.c_uint32, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(Error)]
    lib.ytgpu_groupby_table_update_strings.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                                       C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int32, C.POINTER(Error)]
    lib.ytgpu_groupby_table_result_strings.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(GroupByMultiResult), C.c_void_p, C.c_uint32,
                                                       C.c_void_p, C.c_uint32, C.c_int, C.POINTER(Error)]
    lib.ytgpu_gather_column.argtypes = [C.c_void_p, C.POINTER(ColumnView), C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                        C.POINTER(C.c_uint64), C.c_int, C.POINTER(Error)]
    lib.ytgpu_gather_string_column.argtypes = [C.c_void_p, C.POINTER(StringColumn), C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_int, C.POINTER(Error)]
    lib.ytgpu_order_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(OrderItem), C.c_uint32,
                                     C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64), C.c_int,
                                     C.POINTER(Error)]
    lib.ytgpu_extract_column.argtypes = [C.c_void_p, C.POINTER(RowsetView), C.c_uint32, C.c_uint8, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_int, C.POINTER(Error)]
    lib.ytgpu_block_agg_state_init.argtypes = [C.POINTER(BlockAggState), C.c_uint8, C.c_uint8]
    lib.ytgpu_block_agg_state_init.restype = None
    lib.ytgpu_block_combine_all.argtypes = [C.c_void_p, C.POINTER(ArrowArray), C.c_void_p, C.POINTER(BlockAggState),
                                            C.POINTER(Error)]
    _lib = lib
    return lib


def check(code: int, err: Error) -> None:
    if code != OK:
        raise YtGpuError(code, err.message.decode(errors="replace"), err.cuda_error)


def make_sort_spec(columns):
    """columns: iterable of dicts/tuples (index, width, type, descending, required)."""
    arr = (KeyColumn * len(columns))()
    for i, c in enumerate(columns):
        if isinstance(c, dict):
            idx, width, typ = c["index"], c.get("width", 0), c.get("type", 0)
            desc, req = c.get("descending", 0), c.get("required", 0)
        else:
            idx, width, typ, desc, req = c
        arr[i] = KeyColumn(idx, width, typ, int(bool(desc)), int(bool(req)), 0)
    spec = SortSpec(C.cast(arr, C.POINTER(KeyColumn)), len(columns))
    spec._keepalive = arr
    return spec
