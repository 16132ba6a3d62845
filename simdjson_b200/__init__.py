"""simdjson_b200 -- simdjson's stage 1 (structural indexing + UTF-8 validation), minify and
validate_utf8 as hand-written sm_90a CUDA kernels behind simdjson's own plug-in boundary.

  csrc/            CUDA kernels + the C ABI (include/sjb200.h) -> libsjb200.so
  plugin/          C++ shim: simdjson::implementation / dom_parser_implementation subclasses ("b200")
  implementation   Python mirror of the same two classes over the C ABI (tests, bench)
  corpus           seeded synthetic corpora (SURVEY.md section 8d)

There is no CPU fallback anywhere in this package.
"""
from .capi import (CAPACITY, COMMA_DELIMITED_FINAL, COMMA_DELIMITED_PARTIAL, EMPTY, ERROR_NAMES, JSON_SEQUENCE_FINAL,  # noqa: F401
                   JSON_SEQUENCE_PARTIAL, MEMALLOC, REGULAR, STREAMING_FINAL, STREAMING_PARTIAL, SUCCESS, UNCLOSED_STRING,
                   UNESCAPED_CHARS, UNEXPECTED_ERROR, UNSUPPORTED_ARCHITECTURE, UTF8_ERROR)
from .implementation import (dom_parser_implementation, get_active_implementation, implementation, lib, minify, validate_utf8)  # noqa: F401

__version__ = "0.1.0"
