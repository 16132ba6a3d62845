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
# capi.Doc (sjb200_doc) as a numpy record
_DOC_DTYPE = np.dtype([("d_buf", np.uint64), ("len", np.uint64), ("d_idx", np.uint64), ("n_structural_indexes", np.uint32), ("error", np.int32)])
assert _DOC_DTYPE.itemsize == C.sizeof(capi.Doc) and all(_DOC_DTYPE.fields[f][1] == getattr(capi.Doc, f).offset for f, _ in capi.Doc._fields_)


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

    def __init__(self, device=0, max_depth=1024):
        self._ctx = C.c_void_p()
        self._device = device
        self.max_depth = max_depth  # the stage-2 depth limit (document_errors_device)
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
        # the sjb200_doc array is filled column by column: field by field through ctypes it cost ~1.5 us of host time per
        # document, all of it before the call's first launch
        n = len(d_bufs)
        docs = np.zeros(n, dtype=_DOC_DTYPE)
        docs["d_buf"] = [b.data_ptr() for b in d_bufs]
        docs["len"] = [b.numel() for b in d_bufs]
        docs["d_idx"] = [t.data_ptr() for t in d_idxs]
        rc = lib().sjb200_stage1_dev_batch(self._ctx, docs.ctypes.data_as(C.POINTER(capi.Doc)), n, mode, _stream_ptr(stream))
        if rc != SUCCESS:
            raise RuntimeError("sjb200_stage1_dev_batch failed: " + self.last_cuda_error())
        return list(zip(docs["error"].tolist(), docs["n_structural_indexes"].tolist()))

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

    def at_pointer_device(self, pointers, d_type, d_payload, d_strbuf, string_bytes, d_docs=None, ndocs=None, stream=None):
        """dom::element::at_pointer of every pointer (str or bytes) in every document, on the device (sjb200_at_pointer_dev)
        over the output of tokens_device: d_docs = a document table (sjb200_document_table_dev, int32 pairs
        {index, byte}) and ndocs its entries in use, or None for one document.  Returns (error int32[P, D], index
        int32[P, D]) CUDA tensors: the index is the structural index of the selected value (0xFFFFFFFF, i.e. -1, on an
        error other than a token error).  A failure of the call itself raises."""
        import torch
        enc = [p.encode() if isinstance(p, str) else bytes(p) for p in pointers]
        P = len(enc)
        D = 1 if d_docs is None else (d_docs.numel() * d_docs.element_size() // 8 if ndocs is None else int(ndocs))
        dev = d_type.device
        out = torch.empty((P, max(D, 1), 2), dtype=torch.int32, device=dev)
        bufs = [C.create_string_buffer(e, len(e)) for e in enc]
        ptrs = (C.c_void_p * max(P, 1))(*[C.addressof(b) for b in bufs])
        lens = (C.c_size_t * max(P, 1))(*[len(e) for e in enc])
        n = d_type.numel()
        rc = lib().sjb200_at_pointer_dev(self._ctx, d_type.data_ptr() if n else None, d_payload.data_ptr() if n else None, n,
                                         d_strbuf.data_ptr() if string_bytes else None, string_bytes,
                                         None if d_docs is None else d_docs.data_ptr(), 0 if d_docs is None else D, ptrs, lens, P,
                                         out.data_ptr() if P else None, _stream_ptr(stream))
        if rc != SUCCESS:
            raise RuntimeError(f"sjb200_at_pointer_dev: {capi.ERROR_NAMES.get(rc, rc)} {self.last_cuda_error()}")
        return out[:, :D, 0], out[:, :D, 1]

    def column_device(self, kind, d_type, d_payload, d_strbuf, string_bytes, err, idx, stream=None):
        """one DOM getter (capi.COLUMN_*: get_int64, get_uint64, get_bool, get_string, get_array().size(),
        get_object().size()) on every row of at_pointer_device's (err, idx), or of one pointer's row of them, on the
        device (sjb200_column_dev) over the same tokens.  Returns CUDA tensors shaped like err: (error int32, row_type
        uint8, values) with values int64 (INT64; UINT64 and the sizes as the bits of the uint64) or bool (BOOL); for
        STRING (error, row_type, offsets int64[rows + 1], bytes uint8[offsets[-1]]), the rows in err's row-major order,
        row r being bytes[offsets[r]:offsets[r + 1]].  A failure of the call raises."""
        import torch
        dev = d_type.device
        shape = tuple(err.shape)
        nrows = err.numel()
        # the {error, index} pairs: the at_pointer_device tensors are views of one (..., 2) int32 tensor, used in place
        contiguous_pairs = (err.dtype == idx.dtype == torch.int32 and err.shape == idx.shape and err.stride() == idx.stride()
                            and idx.data_ptr() == err.data_ptr() + 4 and err.is_cuda and idx.is_cuda)
        if contiguous_pairs:
            want, acc = [], 2
            for s in reversed(shape):
                want.append(acc)
                acc *= s
            contiguous_pairs = all(st == w for st, w, s in zip(err.stride(), reversed(want), shape) if s > 1)
        rows = err if contiguous_pairs else torch.stack((err.to(torch.int32), idx.to(torch.int32)), -1).to(dev)
        rows_ptr = rows.data_ptr() if nrows else None
        e = torch.empty(max(nrows, 1), dtype=torch.int32, device=dev)
        t = torch.empty(max(nrows, 1), dtype=torch.uint8, device=dev)
        n = d_type.numel()
        res = capi.ColumnResult()

        def call(values, offsets, d_bytes, cap):
            return lib().sjb200_column_dev(self._ctx, kind, d_type.data_ptr() if n else None, d_payload.data_ptr() if n else None, n,
                                           d_strbuf.data_ptr() if string_bytes else None, string_bytes, rows_ptr, nrows, e.data_ptr(), t.data_ptr(),
                                           values, offsets, d_bytes, cap, C.byref(res), _stream_ptr(stream))

        if kind == capi.COLUMN_STRING:
            offsets = torch.empty(nrows + 1, dtype=torch.int64, device=dev)
            rc = call(None, offsets.data_ptr(), None, 0)
            if rc == capi.CAPACITY:  # the bytes are sized by the first call
                out_bytes = torch.empty(max(res.string_bytes, 1), dtype=torch.uint8, device=dev)
                rc = call(None, offsets.data_ptr(), out_bytes.data_ptr(), res.string_bytes)
            else:
                out_bytes = torch.empty(1, dtype=torch.uint8, device=dev)
            if rc != SUCCESS:
                raise RuntimeError(f"sjb200_column_dev: {capi.ERROR_NAMES.get(rc, rc)} {self.last_cuda_error()}")
            return e[:nrows].view(shape), t[:nrows].view(shape), offsets, out_bytes[: res.string_bytes]
        vals = torch.empty(max(nrows, 1), dtype=torch.bool if kind == capi.COLUMN_BOOL else torch.int64, device=dev)
        rc = call(vals.data_ptr(), None, None, 0)
        if rc != SUCCESS:
            raise RuntimeError(f"sjb200_column_dev: {capi.ERROR_NAMES.get(rc, rc)} {self.last_cuda_error()}")
        return e[:nrows].view(shape), t[:nrows].view(shape), vals[:nrows].view(shape)

    def column_double_device(self, d_buf, d_type, d_payload, err, idx, d_idx=None, stream=None):
        """element::get_double on every row of at_pointer_device's (err, idx), or of one pointer's row of them, on the
        device (sjb200_column_double_dev): d_buf is the input of the stage-1 call whose structurals d_idx holds (default:
        the buffer the last device-resident call wrote) and (d_type, d_payload) its tokens_device output.  Returns CUDA
        tensors shaped like err: (error int32, row_type uint8, values float64), the correctly rounded double of each 'd',
        'l' and 'u' row and +0.0 on an error.  A failure of the call raises."""
        import torch
        dev = d_type.device
        shape = tuple(err.shape)
        nrows = err.numel()
        if d_idx is None:
            d_idx = self.device_index_buffer()
        rows = torch.stack((err.to(torch.int32), idx.to(torch.int32)), -1).to(dev).contiguous()
        e = torch.empty(max(nrows, 1), dtype=torch.int32, device=dev)
        t = torch.empty(max(nrows, 1), dtype=torch.uint8, device=dev)
        v = torch.empty(max(nrows, 1), dtype=torch.float64, device=dev)
        n = d_type.numel()
        res = capi.ColumnResult()
        rc = lib().sjb200_column_double_dev(self._ctx, d_buf.data_ptr() if d_buf.numel() else None, d_buf.numel(), d_idx.data_ptr() if n else None,
                                            d_type.data_ptr() if n else None, d_payload.data_ptr() if n else None, n, rows.data_ptr() if nrows else None,
                                            nrows, e.data_ptr(), t.data_ptr(), v.data_ptr(), C.byref(res), _stream_ptr(stream))
        if rc != SUCCESS:
            raise RuntimeError(f"sjb200_column_double_dev: {capi.ERROR_NAMES.get(rc, rc)} {self.last_cuda_error()}")
        return e[:nrows].view(shape), t[:nrows].view(shape), v[:nrows].view(shape)

    def document_errors_device(self, d_type, d_payload, d_docs=None, ndocs=None, max_depth=None, stream=None):
        """the error stage 2 returns for every document (sjb200_document_errors_dev) over the output of tokens_device:
        d_docs = a document table (sjb200_document_table_dev, int32 pairs {index, byte}) and ndocs its entries in use, or
        None for one document; max_depth defaults to the parser's.  Returns (capi.DocumentErrorsResult, error int32[D],
        index int32[D]) with the results on the device: the index is the structural at which the error was decided, one
        past the document's value on SUCCESS (0xFFFFFFFF, i.e. -1, for a bad table).  A failure of the call raises."""
        import torch
        D = 1 if d_docs is None else (d_docs.numel() * d_docs.element_size() // 8 if ndocs is None else int(ndocs))
        out = torch.empty((max(D, 1), 2), dtype=torch.int32, device=d_type.device)
        res = capi.DocumentErrorsResult()
        n = d_type.numel()
        rc = lib().sjb200_document_errors_dev(self._ctx, d_type.data_ptr() if n else None, d_payload.data_ptr() if n else None, n,
                                              None if d_docs is None else d_docs.data_ptr(), 0 if d_docs is None else D,
                                              self.max_depth if max_depth is None else max_depth, out.data_ptr(), C.byref(res), _stream_ptr(stream))
        if rc != SUCCESS:
            raise RuntimeError(f"sjb200_document_errors_dev: {capi.ERROR_NAMES.get(rc, rc)} {self.last_cuda_error()}")
        return res, out[:D, 0], out[:D, 1]

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
        """-> (error_code, parser or None); L97-101.  max_depth is the default of document_errors_device."""
        p = dom_parser_implementation(self._device, max_depth)
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
