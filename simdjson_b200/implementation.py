"""Host-side mirror of the reference's plug-in interface for the stage-1 path.

The reference is C++, and the C++ shim that plugs into an unmodified simdjson lives in
simdjson_b200/plugin/ (b200_implementation.{h,cpp}).  This module mirrors the same two
classes for Python callers (tests, bench.py) on top of the same C ABI:

  implementation               include/simdjson/implementation.h L45-160
      name(), description(), create_dom_parser_implementation(), minify(), validate_utf8()
  dom_parser_implementation    include/simdjson/internal/dom_parser_implementation.h L48-242
      stage1(buf,len,mode), set_capacity(), n_structural_indexes, structural_indexes,
      next_structural_index, capacity()

Names, argument meaning and error behaviour follow the reference; errors are returned as
simdjson::error_code integers, never raised.  Stage 2 is out of scope (SURVEY.md section 8).
"""
import ctypes as C

import numpy as np

from . import capi
from .capi import (CAPACITY, EMPTY, MEMALLOC, REGULAR, SUCCESS, UNEXPECTED_ERROR, UNSUPPORTED_ARCHITECTURE, UTF8_ERROR)  # noqa: F401

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        _LIB = capi.load()
    return _LIB


def _host_u8(buf):
    if isinstance(buf, np.ndarray):
        return np.ascontiguousarray(buf, dtype=np.uint8)
    return np.frombuffer(bytes(buf), dtype=np.uint8)


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _stream_ptr(stream):
    if stream is None:
        import torch
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if hasattr(stream, "cuda_stream"):
        return C.c_void_p(stream.cuda_stream)
    return C.c_void_p(int(stream))


class dom_parser_implementation:
    """One parser instance = one CUDA context object (own stream and scratch)."""

    def __init__(self, device=0):
        self._ctx = C.c_void_p()
        self._device = device
        self._capacity = 0
        self.n_structural_indexes = 0
        self.structural_indexes = None  # numpy uint32[ROUNDUP(capacity,64)+9] (host calls)
        self.next_structural_index = 0
        self._d_idx = None  # torch uint32-as-int32 tensor for device-resident calls

    # -- lifetime
    def _create(self, capacity):
        rc = lib().sjb200_create(self._device, capacity, C.byref(self._ctx))
        if rc == SUCCESS:
            self._after_capacity(capacity)
        return rc

    def close(self):
        if self._ctx:
            self._unpin()
            lib().sjb200_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def _unpin(self):
        if getattr(self, "_pinned", False) and self.structural_indexes is not None:
            lib().sjb200_unpin_host_memory(self._ctx, self.structural_indexes.ctypes.data)
        self._pinned = False

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _after_capacity(self, capacity):
        self._capacity = capacity
        self._unpin()
        words = lib().sjb200_index_words(capacity)
        self.structural_indexes = np.zeros(words, dtype=np.uint32)
        self.structural_indexes[0] = 0
        # page-lock the index array like the C++ plug-in does, so the D2H of the indexes runs at PCIe speed
        self._pinned = lib().sjb200_pin_host_memory(self._ctx, self.structural_indexes.ctypes.data, words * 4) == SUCCESS
        self.n_structural_indexes = 0
        self._d_idx = None

    def capacity(self):
        return self._capacity

    def set_capacity(self, capacity):
        """generic/dom_parser_implementation.h L66-82: > 0xFFFFFFFF -> CAPACITY; reallocates the index array"""
        rc = lib().sjb200_set_capacity(self._ctx, capacity)
        if rc == SUCCESS:
            self._after_capacity(capacity)
        return rc

    def set_option(self, key, value):
        return lib().sjb200_set_option(self._ctx, key.encode(), int(value))

    def get_stat(self, key):
        return lib().sjb200_get_stat(self._ctx, key.encode())

    def last_cuda_error(self):
        return lib().sjb200_last_cuda_error(self._ctx).decode()

    # -- stage 1, host buffer (what dom::parser / document_stream call)
    def stage1(self, buf, mode=REGULAR):
        a = _host_u8(buf)
        n = C.c_uint32(self.n_structural_indexes)
        ptr = a.ctypes.data if len(a) else None
        rc = lib().sjb200_stage1(self._ctx, ptr, len(a), mode, self.structural_indexes.ctypes.data, C.byref(n))
        self.n_structural_indexes = n.value
        if rc in (SUCCESS, UTF8_ERROR) or (rc == EMPTY and len(a) > 0):
            self.next_structural_index = 0
        return rc

    # -- stage 1, input already in HBM (torch uint8 CUDA tensor); indexes stay on the device
    def device_index_buffer(self, nbytes=None):
        import torch
        if nbytes is None and self._d_idx is not None:
            return self._d_idx  # the buffer the last device-resident call wrote
        words = lib().sjb200_index_words(self._capacity if nbytes is None else nbytes)
        if self._d_idx is None or self._d_idx.numel() < words:
            self._d_idx = torch.empty(words, dtype=torch.int32, device=f"cuda:{self._device}")
        return self._d_idx

    def stage1_device(self, d_buf, mode=REGULAR, d_idx=None, stream=None):
        if d_idx is None:
            d_idx = self.device_index_buffer(d_buf.numel())
        n = C.c_uint32(self.n_structural_indexes)
        rc = lib().sjb200_stage1_dev(self._ctx, d_buf.data_ptr(), d_buf.numel(), mode, d_idx.data_ptr(), C.byref(n), _stream_ptr(stream))
        self.n_structural_indexes = n.value
        return rc

    def stage1_device_batch(self, d_bufs, d_idxs, mode=REGULAR, stream=None):
        """many device-resident documents in one call -> list of (error_code, n_structural_indexes)"""
        n = len(d_bufs)
        docs = (capi.Doc * n)()
        for i in range(n):
            docs[i].d_buf = d_bufs[i].data_ptr()
            docs[i].len = d_bufs[i].numel()
            docs[i].d_idx = d_idxs[i].data_ptr()
            docs[i].n_structural_indexes = 0
        rc = lib().sjb200_stage1_dev_batch(self._ctx, docs, n, mode, _stream_ptr(stream))
        if rc != SUCCESS:
            raise RuntimeError("sjb200_stage1_dev_batch failed: " + self.last_cuda_error())
        return [(docs[i].error, docs[i].n_structural_indexes) for i in range(n)]

    def stage1_device_enqueue(self, d_buf, mode=REGULAR, d_idx=None, stream=None):
        if d_idx is None:
            d_idx = self.device_index_buffer(d_buf.numel())
        return lib().sjb200_stage1_dev_enqueue(self._ctx, d_buf.data_ptr(), d_buf.numel(), mode, d_idx.data_ptr(), _stream_ptr(stream))

    def stage1_device_finish(self):
        n = C.c_uint32(self.n_structural_indexes)
        rc = lib().sjb200_stage1_dev_finish(self._ctx, C.byref(n))
        self.n_structural_indexes = n.value
        return rc

    def tokens_device(self, d_buf, d_idx=None, n=None, strbuf_capacity=None, stream=None):
        """stage-2-lite (sjb200_tokens_dev) on the output of the last device-resident stage-1 call: returns
        (capi.TokensResult, d_type uint8[n], d_payload int64[n] (bit pattern of the uint64), d_strbuf uint8[capacity])"""
        import torch
        if d_idx is None:
            d_idx = self.device_index_buffer()
        if n is None:
            n = self.n_structural_indexes
        cap = lib().sjb200_string_buf_capacity(d_buf.numel()) if strbuf_capacity is None else strbuf_capacity
        dev = d_buf.device
        d_type = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        d_payload = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        d_strbuf = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        res = capi.TokensResult()
        lib().sjb200_tokens_dev(self._ctx, d_buf.data_ptr(), d_buf.numel(), d_idx.data_ptr(), n, d_type.data_ptr(), d_payload.data_ptr(),
                                d_strbuf.data_ptr() if cap else None, cap, C.byref(res), _stream_ptr(stream))
        return res, d_type[:n], d_payload[:n], d_strbuf

    def stage1_shard_device(self, d_buf, state_in=0, last_shard=True, d_idx=None, stream=None):
        """one GPU's piece of a sharded scan; returns (error_code, capi.ShardResult)"""
        if d_idx is None:
            d_idx = self.device_index_buffer(d_buf.numel())
        res = capi.ShardResult()
        rc = lib().sjb200_stage1_shard_dev(self._ctx, d_buf.data_ptr(), d_buf.numel(), state_in, int(last_shard), d_idx.data_ptr(),
                                           C.byref(res), _stream_ptr(stream))
        return rc, res

    def stage1_shard_device_enqueue(self, d_buf, d_result, d_idx=None, stream=None):
        """speculative shard pass, no host sync: d_result = 3 x int64 device tensor {count, state|ttable<<32, flags}"""
        if d_idx is None:
            d_idx = self.device_index_buffer(d_buf.numel())
        return lib().sjb200_stage1_shard_dev_enqueue(self._ctx, d_buf.data_ptr(), d_buf.numel(), d_idx.data_ptr(), d_result.data_ptr(),
                                                     _stream_ptr(stream))

    # -- minify / utf8 on this parser's context (the reference routes them through `implementation`)
    def _minify_host(self, buf):
        a = _host_u8(buf)
        dst = np.empty(max(len(a), 1), dtype=np.uint8)  # exactly len bytes, like tests/dom/basictests.cpp L1916
        dl = C.c_size_t(0)
        rc = lib().sjb200_minify(self._ctx, a.ctypes.data if len(a) else None, len(a), dst.ctypes.data, C.byref(dl))
        return rc, dst[: dl.value]

    def _validate_utf8_host(self, buf):
        a = _host_u8(buf)
        return bool(lib().sjb200_validate_utf8(self._ctx, a.ctypes.data if len(a) else None, len(a)))

    def minify_device(self, d_buf, d_dst, stream=None):
        dl = C.c_size_t(0)
        rc = lib().sjb200_minify_dev(self._ctx, d_buf.data_ptr(), d_buf.numel(), d_dst.data_ptr(), C.byref(dl), _stream_ptr(stream))
        return rc, dl.value

    def minify_device_enqueue(self, d_buf, d_dst, stream=None):
        return lib().sjb200_minify_dev_enqueue(self._ctx, d_buf.data_ptr(), d_buf.numel(), d_dst.data_ptr(), _stream_ptr(stream))

    def minify_device_finish(self):
        dl = C.c_size_t(0)
        rc = lib().sjb200_minify_dev_finish(self._ctx, C.byref(dl))
        return rc, dl.value

    def validate_utf8_device(self, d_buf, stream=None):
        return lib().sjb200_validate_utf8_dev(self._ctx, d_buf.data_ptr(), d_buf.numel(), _stream_ptr(stream))

    def validate_utf8_device_enqueue(self, d_buf, stream=None):
        return lib().sjb200_validate_utf8_dev_enqueue(self._ctx, d_buf.data_ptr(), d_buf.numel(), _stream_ptr(stream))

    def validate_utf8_device_finish(self):
        return lib().sjb200_validate_utf8_dev_finish(self._ctx)


class implementation:
    """simdjson::implementation for the H100 (include/simdjson/implementation.h L45-160)."""

    def __init__(self, device=0):
        self._device = device
        self._util = None  # lazily created context for the stateless minify / validate_utf8 calls

    def name(self):
        return "b200"

    def description(self):
        return "NVIDIA H100 (sm_90a) stage 1"

    def required_instruction_sets(self):
        return 0

    def supported_by_runtime_system(self):
        p = dom_parser_implementation(self._device)
        rc = p._create(0)
        p.close()
        return rc == SUCCESS

    def create_dom_parser_implementation(self, capacity, max_depth=1024):
        """-> (error_code, parser or None); L97-101"""
        _ = max_depth  # stage 2 stacks are not part of this path
        p = dom_parser_implementation(self._device)
        rc = p._create(capacity)
        return (rc, p) if rc == SUCCESS else (rc, None)

    def _utility(self):
        if self._util is None:
            rc, p = self.create_dom_parser_implementation(0)
            if rc != SUCCESS:
                raise RuntimeError(f"sjb200_create failed: {capi.ERROR_NAMES.get(rc, rc)}")
            self._util = p
        return self._util

    def minify(self, buf):
        """-> (error_code, minified bytes as numpy uint8); L116"""
        return self._utility()._minify_host(buf)

    def validate_utf8(self, buf):
        """-> bool; L128"""
        return self._utility()._validate_utf8_host(buf)


_ACTIVE = {}


def get_active_implementation(device=0):
    """src/implementation.cpp L321-332 (there is exactly one implementation here)."""
    if device not in _ACTIVE:
        _ACTIVE[device] = implementation(device)
    return _ACTIVE[device]


def minify(buf, device=0):
    """simdjson::minify(buf,len,dst,dst_len) -- src/implementation.cpp L334-336"""
    return get_active_implementation(device).minify(buf)


def validate_utf8(buf, device=0):
    """simdjson::validate_utf8(buf,len) -- src/implementation.cpp L337-339"""
    return get_active_implementation(device).validate_utf8(buf)
