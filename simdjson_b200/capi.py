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
    "sjb200_stage1", "sjb200_minify", "sjb200_validate_utf8",
    "sjb200_stage1_dev", "sjb200_minify_dev", "sjb200_validate_utf8_dev", "sjb200_stage1_dev_batch",
    "sjb200_document_table_dev", "sjb200_stage1_dev_enqueue", "sjb200_stage1_dev_finish", "sjb200_minify_dev_enqueue", "sjb200_minify_dev_finish",
    "sjb200_validate_utf8_dev_enqueue", "sjb200_validate_utf8_dev_finish",
    "sjb200_stage1_shard_dev", "sjb200_stage1_shard_dev_enqueue", "sjb200_fold_state", "sjb200_shard_cut", "sjb200_shard_cut_line",
    "sjb200_comm_create", "sjb200_comm_destroy", "sjb200_comm_get_handle", "sjb200_comm_connect", "sjb200_comm_connect_local",
    "sjb200_stage1_sharded", "sjb200_stage1_sharded_enqueue", "sjb200_stage1_sharded_finish",
    "sjb200_tokens_dev", "sjb200_string_buf_capacity",
]
COMM_HANDLE_BYTES = 64

# simdjson::error_code values of this path (include/simdjson/error.h L19-54)
SUCCESS, CAPACITY, MEMALLOC, UTF8_ERROR, EMPTY, UNESCAPED_CHARS, UNCLOSED_STRING, UNSUPPORTED_ARCHITECTURE, UNEXPECTED_ERROR = 0, 1, 2, 11, 13, 14, 15, 16, 24
ERROR_NAMES = {0: "SUCCESS", 1: "CAPACITY", 2: "MEMALLOC", 3: "TAPE_ERROR", 5: "STRING_ERROR", 6: "T_ATOM_ERROR", 7: "F_ATOM_ERROR", 8: "N_ATOM_ERROR",
               9: "NUMBER_ERROR", 10: "BIGINT_ERROR", 11: "UTF8_ERROR", 13: "EMPTY", 14: "UNESCAPED_CHARS", 15: "UNCLOSED_STRING",
               16: "UNSUPPORTED_ARCHITECTURE", 24: "UNEXPECTED_ERROR"}

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
        "sjb200_tokens_dev": (C.c_int, [vp, vp, sz, vp, C.c_uint32, vp, vp, vp, sz, C.POINTER(TokensResult), vp]),
        "sjb200_string_buf_capacity": (sz, [sz]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _ = u8p
    return L
