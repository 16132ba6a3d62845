"""ctypes binding of the C ABI (include/sjb200.h) exported by simdjson_b200/libsjb200.so.

The library is the product: this module only loads it.  There is no Python or CPU
fallback -- if the shared object is missing the import fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SJB200_LIB") or os.path.join(_HERE, "libsjb200.so")  # SJB200_LIB: build variants for tuning

# every symbol include/sjb200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "sjb200_create", "sjb200_destroy", "sjb200_set_capacity", "sjb200_capacity", "sjb200_index_words", "sjb200_device",
    "sjb200_last_cuda_error", "sjb200_set_option", "sjb200_get_stat", "sjb200_pin_host_memory", "sjb200_unpin_host_memory", "sjb200_get_debug_timeline",
    "sjb200_get_launch_stamps",
    "sjb200_stage1", "sjb200_minify", "sjb200_validate_utf8",
    "sjb200_stage1_dev", "sjb200_minify_dev", "sjb200_validate_utf8_dev", "sjb200_stage1_dev_batch",
    "sjb200_document_table_dev", "sjb200_stage1_dev_enqueue", "sjb200_stage1_dev_finish", "sjb200_minify_dev_enqueue", "sjb200_minify_dev_finish",
    "sjb200_validate_utf8_dev_enqueue", "sjb200_validate_utf8_dev_finish",
    "sjb200_stage1_shard_dev", "sjb200_stage1_shard_dev_enqueue", "sjb200_fold_state", "sjb200_shard_cut", "sjb200_shard_cut_line",
    "sjb200_comm_create", "sjb200_comm_destroy", "sjb200_comm_get_handle", "sjb200_comm_connect", "sjb200_comm_connect_local",
    "sjb200_stage1_sharded", "sjb200_stage1_sharded_enqueue", "sjb200_stage1_sharded_finish",
    "sjb200_minify_sharded", "sjb200_minify_sharded_enqueue", "sjb200_minify_sharded_finish",
    "sjb200_validate_utf8_sharded", "sjb200_validate_utf8_sharded_enqueue", "sjb200_validate_utf8_sharded_finish",
    "sjb200_tokens_dev", "sjb200_string_buf_capacity",
    "sjb200_stage1_sharded_stream", "sjb200_stage1_sharded_stream_enqueue", "sjb200_stage1_sharded_stream_finish",
    "sjb200_document_table_shard_dev", "sjb200_stream_fold",
    "sjb200_stage1_sharded_delimited", "sjb200_stage1_sharded_delimited_enqueue", "sjb200_stage1_sharded_delimited_finish", "sjb200_delimited_fold",
    "sjb200_tokens_sharded", "sjb200_tokens_sharded_enqueue", "sjb200_tokens_sharded_finish",
    "sjb200_at_pointer_dev", "sjb200_document_errors_dev",
    "sjb200_document_errors_sharded", "sjb200_document_errors_sharded_enqueue", "sjb200_document_errors_sharded_finish",
    "sjb200_grammar_edge_fold", "sjb200_grammar_result_fold",
    "sjb200_at_pointer_sharded", "sjb200_at_pointer_sharded_enqueue", "sjb200_at_pointer_sharded_finish", "sjb200_pointer_edge_fold",
    "sjb200_column_dev", "sjb200_column_double_dev",
]
COMM_HANDLE_BYTES = 64

# simdjson::error_code values of this path (include/simdjson/error.h L19-54)
SUCCESS, CAPACITY, MEMALLOC, UTF8_ERROR, EMPTY, UNESCAPED_CHARS, UNCLOSED_STRING, UNSUPPORTED_ARCHITECTURE, UNEXPECTED_ERROR = 0, 1, 2, 11, 13, 14, 15, 16, 24
ERROR_NAMES = {0: "SUCCESS", 1: "CAPACITY", 2: "MEMALLOC", 3: "TAPE_ERROR", 4: "DEPTH_ERROR", 5: "STRING_ERROR", 6: "T_ATOM_ERROR", 7: "F_ATOM_ERROR", 8: "N_ATOM_ERROR",
               9: "NUMBER_ERROR", 10: "BIGINT_ERROR", 11: "UTF8_ERROR", 13: "EMPTY", 14: "UNESCAPED_CHARS", 15: "UNCLOSED_STRING",
               16: "UNSUPPORTED_ARCHITECTURE", 17: "INCORRECT_TYPE", 18: "NUMBER_OUT_OF_RANGE", 19: "INDEX_OUT_OF_BOUNDS", 20: "NO_SUCH_FIELD", 22: "INVALID_JSON_POINTER",
               24: "UNEXPECTED_ERROR"}
INCORRECT_TYPE, INDEX_OUT_OF_BOUNDS, NO_SUCH_FIELD, INVALID_JSON_POINTER = 17, 19, 20, 22
NUMBER_OUT_OF_RANGE = 18
NUMBER_ERROR = 9
# kinds of sjb200_column_dev (SJB200_COLUMN_*)
COLUMN_INT64, COLUMN_UINT64, COLUMN_BOOL, COLUMN_STRING, COLUMN_ARRAY_SIZE, COLUMN_OBJECT_SIZE = 1, 2, 3, 4, 5, 6
DEPTH_ERROR = 4
# the deepest max_depth sjb200_document_errors_dev accepts (SJB200_DOCUMENT_MAX_DEPTH)
DOCUMENT_MAX_DEPTH = 4096
# limits of sjb200_at_pointer_dev (SJB200_POINTER_MAX_*)
POINTER_MAX_POINTERS, POINTER_MAX_TOKENS, POINTER_MAX_BYTES = 65536, 1024, 1 << 20

# simdjson::stage1_mode (include/simdjson/internal/dom_parser_implementation.h L22-27)
REGULAR, STREAMING_PARTIAL, STREAMING_FINAL, JSON_SEQUENCE_PARTIAL, JSON_SEQUENCE_FINAL, COMMA_DELIMITED_PARTIAL, COMMA_DELIMITED_FINAL = range(7)


class Doc(C.Structure):
    _fields_ = [("d_buf", C.c_void_p), ("len", C.c_size_t), ("d_idx", C.c_void_p), ("n_structural_indexes", C.c_uint32), ("error", C.c_int)]


class TokensResult(C.Structure):
    _fields_ = [("error", C.c_int), ("first_error_index", C.c_uint32), ("n_strings", C.c_uint32), ("string_bytes", C.c_uint64)]


class ShardResult(C.Structure):
    _fields_ = [("ttable", C.c_uint32), ("state_out", C.c_uint32), ("flags", C.c_uint32), ("reserved", C.c_uint32), ("count", C.c_uint64)]


class ShardedResult(C.Structure):
    _fields_ = [("count", C.c_uint64), ("base", C.c_uint64), ("total_count", C.c_uint64), ("state_in", C.c_uint32), ("state_out", C.c_uint32),
                ("final_state", C.c_uint32), ("flags", C.c_uint32), ("flags_all", C.c_uint32), ("rescanned", C.c_uint32)]


class ShardedStreamResult(C.Structure):
    _fields_ = [("shard", ShardedResult), ("n", C.c_uint64), ("kept", C.c_uint64), ("bytes_before", C.c_uint64), ("total_bytes", C.c_uint64),
                ("first_starts_document", C.c_uint32), ("reserved", C.c_uint32)]


class StreamSummary(C.Structure):
    _fields_ = [("count", C.c_uint64), ("len", C.c_uint32), ("first_byte", C.c_uint32), ("last_byte", C.c_uint32), ("start_index", C.c_uint32),
                ("start_byte", C.c_uint32), ("net_obj", C.c_int32), ("net_arr", C.c_int32), ("role_first", C.c_uint32), ("role_last", C.c_uint32),
                ("has_start", C.c_uint32)]


class StreamRank(C.Structure):
    _fields_ = [("kept", C.c_uint64), ("bytes_before", C.c_uint64), ("first_starts_document", C.c_uint32), ("nrewrites", C.c_uint32),
                ("rewrite_pos", C.c_uint32 * 2), ("rewrite_val", C.c_uint32 * 2)]


class StreamFoldResult(C.Structure):
    _fields_ = [("error", C.c_int), ("n_written", C.c_uint32), ("n", C.c_uint64), ("total_bytes", C.c_uint64)]


class ShardedDelimitedResult(C.Structure):
    _fields_ = [("stream", ShardedStreamResult), ("filtered", C.c_uint64), ("filtered_before", C.c_uint64), ("tail", C.c_uint32 * 3),
                ("reserved", C.c_uint32)]


class DelimitedSummary(C.Structure):
    _fields_ = [("count", C.c_uint64), ("len", C.c_uint32), ("filtered", C.c_uint32), ("seps", C.c_uint32), ("last_sep", C.c_uint32),
                ("below", C.c_uint32), ("reserved", C.c_uint32), ("walk", StreamSummary), ("walk_below", StreamSummary)]


class DelimitedRank(C.Structure):
    _fields_ = [("kept", C.c_uint64), ("filtered_before", C.c_uint64), ("bytes_before", C.c_uint64), ("first_starts_document", C.c_uint32),
                ("reserved", C.c_uint32)]


class DelimitedFoldResult(C.Structure):
    _fields_ = [("error", C.c_int), ("n_written", C.c_uint32), ("n", C.c_uint64), ("total_bytes", C.c_uint64), ("tail_rank", C.c_int32 * 3),
                ("tail_pos", C.c_uint32 * 3), ("tail_filtered", C.c_uint32 * 3), ("tail_val", C.c_uint32 * 3)]


class ShardedTokensResult(C.Structure):
    _fields_ = [("error", C.c_int), ("dirty_cuts", C.c_uint32), ("short_ranks", C.c_uint32), ("reserved", C.c_uint32),
                ("first_error_index", C.c_uint64), ("tokens_before", C.c_uint64), ("bytes_before", C.c_uint64), ("n_strings", C.c_uint64),
                ("strings_before", C.c_uint64), ("total_strings", C.c_uint64), ("string_bytes", C.c_uint64), ("string_base", C.c_uint64),
                ("total_string_bytes", C.c_uint64)]


class PointerResult(C.Structure):
    _fields_ = [("error", C.c_int32), ("index", C.c_uint32)]


class ColumnResult(C.Structure):
    _fields_ = [("rows_in_error", C.c_uint32), ("reserved", C.c_uint32), ("string_bytes", C.c_uint64)]


class DocumentErrorsResult(C.Structure):
    _fields_ = [("ndocs_in_error", C.c_uint32), ("first_doc_in_error", C.c_uint32)]


class ShardedDocumentError(C.Structure):
    _fields_ = [("error", C.c_int32), ("reserved", C.c_uint32), ("index", C.c_uint64)]


class ShardedDocumentErrorsResult(C.Structure):
    _fields_ = [("error", C.c_int), ("first_error", C.c_int32), ("docs_before", C.c_uint64), ("tokens_before", C.c_uint64), ("ndocs", C.c_uint64),
                ("ndocs_in_error", C.c_uint64), ("first_doc_in_error", C.c_uint64), ("first_error_index", C.c_uint64)]


class GrammarEdge(C.Structure):
    _fields_ = [("n", C.c_uint32), ("ndocs", C.c_uint32), ("flags", C.c_uint32), ("max_depth", C.c_uint32), ("types", C.c_uint32), ("first_start", C.c_uint32)]


class GrammarRank(C.Structure):
    _fields_ = [("tokens_before", C.c_uint64), ("docs_before", C.c_uint64), ("owned", C.c_uint32), ("holds_root", C.c_uint32), ("halo_before", C.c_uint32),
                ("halo_after", C.c_uint32), ("halo_flags", C.c_uint32), ("last_type", C.c_uint32)]


class GrammarEdgeFoldResult(C.Structure):
    _fields_ = [("error", C.c_int), ("bad_table", C.c_uint32), ("n", C.c_uint64), ("ndocs", C.c_uint64)]


class GrammarTally(C.Structure):
    _fields_ = [("lead", C.c_uint64), ("last", C.c_uint64), ("first_key", C.c_uint64), ("errors", C.c_uint32), ("first_doc", C.c_uint32)]


class ShardedPointerResult(C.Structure):
    _fields_ = [("error", C.c_int32), ("reserved", C.c_uint32), ("index", C.c_uint64)]


class ShardedPointerSummary(C.Structure):
    _fields_ = [("error", C.c_int), ("rounds", C.c_uint32), ("docs_before", C.c_uint64), ("tokens_before", C.c_uint64), ("ndocs", C.c_uint64),
                ("walks_forwarded", C.c_uint64)]


class PointerEdge(C.Structure):
    _fields_ = [("n", C.c_uint32), ("ndocs", C.c_uint32), ("flags", C.c_uint32), ("npointers", C.c_uint32), ("hash", C.c_uint64), ("types", C.c_uint32),
                ("first_entry", C.c_uint32), ("lead_error_index", C.c_uint32), ("lead_error", C.c_uint32)]


class PointerRank(C.Structure):
    _fields_ = [("tokens_before", C.c_uint64), ("docs_before", C.c_uint64), ("owned", C.c_uint32), ("walks", C.c_uint32), ("prev_holder", C.c_int32),
                ("next_holder", C.c_int32), ("next_type", C.c_uint32), ("lead_owner", C.c_int32), ("tail_owner", C.c_int32), ("tail_continues", C.c_uint32),
                ("tail_through", C.c_int32), ("tail_error", C.c_uint32), ("tail_after", C.c_uint64), ("tail_error_index", C.c_uint64)]


class PointerEdgeFoldResult(C.Structure):
    _fields_ = [("error", C.c_int), ("bad_table", C.c_uint32), ("n", C.c_uint64), ("ndocs", C.c_uint64)]


def load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  simdjson_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    u8p, u32p, vp, sz = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.c_void_p, C.c_size_t
    sig = {
        "sjb200_create": (C.c_int, [C.c_int, sz, C.POINTER(vp)]),
        "sjb200_destroy": (None, [vp]),
        "sjb200_set_capacity": (C.c_int, [vp, sz]),
        "sjb200_capacity": (sz, [vp]),
        "sjb200_index_words": (sz, [sz]),
        "sjb200_device": (C.c_int, [vp]),
        "sjb200_last_cuda_error": (C.c_char_p, [vp]),
        "sjb200_set_option": (C.c_int, [vp, C.c_char_p, C.c_long]),
        "sjb200_get_stat": (C.c_double, [vp, C.c_char_p]),
        "sjb200_get_debug_timeline": (C.c_long, [vp, vp, sz]),
        "sjb200_get_launch_stamps": (C.c_long, [vp, vp, sz]),
        "sjb200_pin_host_memory": (C.c_int, [vp, vp, sz]),
        "sjb200_unpin_host_memory": (C.c_int, [vp, vp]),
        "sjb200_stage1": (C.c_int, [vp, vp, sz, C.c_int, vp, u32p]),
        "sjb200_minify": (C.c_int, [vp, vp, sz, vp, C.POINTER(sz)]),
        "sjb200_validate_utf8": (C.c_int, [vp, vp, sz]),
        "sjb200_stage1_dev": (C.c_int, [vp, vp, sz, C.c_int, vp, u32p, vp]),
        "sjb200_minify_dev": (C.c_int, [vp, vp, sz, vp, C.POINTER(sz), vp]),
        "sjb200_validate_utf8_dev": (C.c_int, [vp, vp, sz, vp]),
        "sjb200_stage1_dev_batch": (C.c_int, [vp, C.POINTER(Doc), C.c_int, C.c_int, vp]),
        "sjb200_document_table_dev": (C.c_int, [vp, vp, vp, C.c_uint32, vp, C.c_uint32, u32p, vp]),
        "sjb200_stage1_dev_enqueue": (C.c_int, [vp, vp, sz, C.c_int, vp, vp]),
        "sjb200_stage1_dev_finish": (C.c_int, [vp, u32p]),
        "sjb200_minify_dev_enqueue": (C.c_int, [vp, vp, sz, vp, vp]),
        "sjb200_minify_dev_finish": (C.c_int, [vp, C.POINTER(sz)]),
        "sjb200_validate_utf8_dev_enqueue": (C.c_int, [vp, vp, sz, vp]),
        "sjb200_validate_utf8_dev_finish": (C.c_int, [vp]),
        "sjb200_stage1_shard_dev": (C.c_int, [vp, vp, sz, C.c_uint32, C.c_int, vp, C.POINTER(ShardResult), vp]),
        "sjb200_stage1_shard_dev_enqueue": (C.c_int, [vp, vp, sz, vp, vp, vp]),
        "sjb200_fold_state": (C.c_uint32, [u32p, C.c_int]),
        "sjb200_shard_cut": (sz, [vp, sz, sz]),
        "sjb200_shard_cut_line": (sz, [vp, sz, sz, sz]),
        "sjb200_comm_create": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(vp)]),
        "sjb200_comm_destroy": (None, [vp]),
        "sjb200_comm_get_handle": (C.c_int, [vp, vp]),
        "sjb200_comm_connect": (C.c_int, [vp, vp]),
        "sjb200_comm_connect_local": (C.c_int, [vp, C.POINTER(vp)]),
        "sjb200_stage1_sharded": (C.c_int, [vp, vp, sz, C.c_int, vp, C.POINTER(ShardedResult), vp]),
        "sjb200_stage1_sharded_enqueue": (C.c_int, [vp, vp, sz, C.c_int, vp, vp]),
        "sjb200_stage1_sharded_finish": (C.c_int, [vp, C.POINTER(ShardedResult)]),
        "sjb200_minify_sharded": (C.c_int, [vp, vp, sz, vp, C.POINTER(ShardedResult), vp]),
        "sjb200_minify_sharded_enqueue": (C.c_int, [vp, vp, sz, vp, vp]),
        "sjb200_minify_sharded_finish": (C.c_int, [vp, C.POINTER(ShardedResult)]),
        "sjb200_validate_utf8_sharded": (C.c_int, [vp, vp, sz, C.POINTER(ShardedResult), vp]),
        "sjb200_validate_utf8_sharded_enqueue": (C.c_int, [vp, vp, sz, vp]),
        "sjb200_validate_utf8_sharded_finish": (C.c_int, [vp, C.POINTER(ShardedResult)]),
        "sjb200_tokens_dev": (C.c_int, [vp, vp, sz, vp, C.c_uint32, vp, vp, vp, sz, C.POINTER(TokensResult), vp]),
        "sjb200_string_buf_capacity": (sz, [sz]),
        "sjb200_stage1_sharded_stream": (C.c_int, [vp, vp, sz, C.c_int, C.c_int, vp, C.POINTER(ShardedStreamResult), vp]),
        "sjb200_stage1_sharded_stream_enqueue": (C.c_int, [vp, vp, sz, C.c_int, C.c_int, vp, vp]),
        "sjb200_stage1_sharded_stream_finish": (C.c_int, [vp, C.POINTER(ShardedStreamResult)]),
        "sjb200_document_table_shard_dev": (C.c_int, [vp, vp, vp, C.c_uint32, C.c_int, vp, C.c_uint32, u32p, vp]),
        "sjb200_stream_fold": (C.c_int, [C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.POINTER(StreamSummary), C.POINTER(StreamFoldResult),
                                         C.POINTER(StreamRank)]),
        "sjb200_stage1_sharded_delimited": (C.c_int, [vp, vp, sz, C.c_int, C.c_int, vp, C.POINTER(ShardedDelimitedResult), vp]),
        "sjb200_stage1_sharded_delimited_enqueue": (C.c_int, [vp, vp, sz, C.c_int, C.c_int, vp, vp]),
        "sjb200_stage1_sharded_delimited_finish": (C.c_int, [vp, C.POINTER(ShardedDelimitedResult)]),
        "sjb200_delimited_fold": (C.c_int, [C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.POINTER(DelimitedSummary), C.POINTER(DelimitedFoldResult),
                                            C.POINTER(DelimitedRank)]),
        "sjb200_tokens_sharded": (C.c_int, [vp, vp, sz, C.c_uint32, vp, C.c_uint32, vp, vp, vp, sz, C.POINTER(ShardedTokensResult), vp]),
        "sjb200_tokens_sharded_enqueue": (C.c_int, [vp, vp, sz, C.c_uint32, vp, C.c_uint32, vp, vp, vp, sz, vp]),
        "sjb200_tokens_sharded_finish": (C.c_int, [vp, C.POINTER(ShardedTokensResult)]),
        "sjb200_at_pointer_dev": (C.c_int, [vp, vp, vp, C.c_uint32, vp, sz, vp, C.c_uint32, vp, vp, C.c_int, vp, vp]),
        "sjb200_document_errors_dev": (C.c_int, [vp, vp, vp, C.c_uint32, vp, C.c_uint32, sz, vp, C.POINTER(DocumentErrorsResult), vp]),
        "sjb200_document_errors_sharded": (C.c_int, [vp, vp, vp, C.c_uint32, C.c_int, vp, C.c_uint32, sz, vp, C.POINTER(ShardedDocumentErrorsResult), vp]),
        "sjb200_document_errors_sharded_enqueue": (C.c_int, [vp, vp, vp, C.c_uint32, C.c_int, vp, C.c_uint32, sz, vp, vp]),
        "sjb200_document_errors_sharded_finish": (C.c_int, [vp, C.POINTER(ShardedDocumentErrorsResult)]),
        "sjb200_grammar_edge_fold": (C.c_int, [C.c_int, C.POINTER(GrammarEdge), C.POINTER(GrammarEdgeFoldResult), C.POINTER(GrammarRank)]),
        "sjb200_grammar_result_fold": (C.c_int, [C.c_int, C.POINTER(GrammarEdge), C.POINTER(GrammarTally), C.POINTER(ShardedDocumentErrorsResult),
                                                 C.POINTER(ShardedDocumentError)]),
        "sjb200_at_pointer_sharded": (C.c_int, [vp, vp, vp, C.c_uint32, vp, sz, C.c_int, vp, C.c_uint32, vp, vp, C.c_int, vp,
                                                C.POINTER(ShardedPointerSummary), vp]),
        "sjb200_at_pointer_sharded_enqueue": (C.c_int, [vp, vp, vp, C.c_uint32, vp, sz, C.c_int, vp, C.c_uint32, vp, vp, C.c_int, vp, vp]),
        "sjb200_at_pointer_sharded_finish": (C.c_int, [vp, C.POINTER(ShardedPointerSummary)]),
        "sjb200_pointer_edge_fold": (C.c_int, [C.c_int, C.POINTER(PointerEdge), C.POINTER(PointerEdgeFoldResult), C.POINTER(PointerRank)]),
        "sjb200_column_dev": (C.c_int, [vp, C.c_int, vp, vp, C.c_uint32, vp, sz, vp, C.c_uint32, vp, vp, vp, vp, vp, sz, C.POINTER(ColumnResult), vp]),
        "sjb200_column_double_dev": (C.c_int, [vp, vp, sz, vp, vp, vp, C.c_uint32, vp, C.c_uint32, vp, vp, vp, C.POINTER(ColumnResult), vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _ = u8p
    return L
