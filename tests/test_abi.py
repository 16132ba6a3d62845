"""The C-ABI library loads and exports every symbol include/sjb200.h declares (no GPU needed)."""
import ctypes as C
import os
import re

import simdjson_b200 as sj
from simdjson_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_header_symbols():
    header = open(os.path.join(ROOT, "include", "sjb200.h")).read()
    declared = sorted(set(re.findall(r"SJB200_API[^;(]*?\b(sjb200_\w+)\s*\(", header)))
    assert len(declared) >= 20
    assert sorted(capi.EXPORTS) == declared
    L = C.CDLL(capi.LIB_PATH)
    for name in declared:
        assert hasattr(L, name), name


def test_error_and_mode_constants_match_header():
    header = open(os.path.join(ROOT, "include", "sjb200.h")).read()
    vals = dict(re.findall(r"SJB200_(\w+) = (\d+)", header))
    assert int(vals["UTF8_ERROR"]) == sj.UTF8_ERROR == 11
    assert int(vals["UNCLOSED_STRING"]) == sj.UNCLOSED_STRING == 15
    assert int(vals["UNSUPPORTED_ARCHITECTURE"]) == sj.UNSUPPORTED_ARCHITECTURE == 16
    assert int(vals["COMMA_DELIMITED_FINAL"]) == sj.COMMA_DELIMITED_FINAL == 6


def test_pure_host_helpers():
    L = capi.load()
    assert L.sjb200_index_words(0) == 9
    assert L.sjb200_index_words(1) == 73
    assert L.sjb200_index_words(64) == 73
    assert L.sjb200_index_words(65) == 137
    # fold of transducers: identity-like chunk (no quotes, ends on whitespace) keeps the state
    tt = (C.c_uint32 * 2)(0b000000, 0b010010)  # second chunk has odd quote parity for both e
    assert L.sjb200_fold_state(tt, 1) == 0
    assert L.sjb200_fold_state(tt, 2) == 0b010
    buf = b"ab\xe2\x82\xacxy"
    p = C.create_string_buffer(buf, len(buf))
    assert L.sjb200_shard_cut(C.addressof(p), len(buf), 3) == 2  # inside the 3-byte char -> back to its lead
    assert L.sjb200_shard_cut(C.addressof(p), len(buf), 5) == 5
    assert L.sjb200_shard_cut(C.addressof(p), len(buf), 99) == len(buf)


def test_no_cpu_fallback_without_gpu():
    """Without a usable sm_90 device the product must fail loudly, not fall back."""
    import torch
    if torch.cuda.is_available():
        return
    impl = sj.get_active_implementation()
    rc, parser = impl.create_dom_parser_implementation(1 << 20)
    assert rc == sj.UNSUPPORTED_ARCHITECTURE and parser is None
    assert impl.supported_by_runtime_system() is False
