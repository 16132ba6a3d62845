"""Multi-GPU sharding of one stage-1 scan (SURVEY.md section 8e): the host-side protocol around
`sjb200_stage1_shard_dev`, and `Comm`, the per-rank object of the sharded stage-1 / minify / validate_utf8 / stage-2-lite
passes whose exchange is fused into the kernels.

Every rank scans its byte range with a *speculated* incoming scanner state (0 = outside a string, no pending
escape, previous byte not a scalar).  A shard's 6-bit carry transducer does not depend on the incoming state, so
one all-gather of {transducer, count, flags} per rank tells every rank everybody's true incoming state; a rank
whose speculation was wrong scans again with the true state and a second all-gather republishes the counts.
Indexes stay shard-relative (uint32) plus a 64-bit base, like document_stream's batch_start + structural_indexes[i]
(include/simdjson/dom/document_stream-inl.h L250).
"""
import collections
import ctypes as C

import numpy as np

from .implementation import lib as _lib


def fold_states(ttables):
    """true incoming state of every shard from the shards' transducers (document starts in state 0)"""
    L = _lib()
    arr = (C.c_uint32 * len(ttables))(*[int(t) for t in ttables])
    return [int(L.sjb200_fold_state(arr, r)) for r in range(len(ttables))]


def fold_stream(mode, final_state, flags_all, summaries):
    """sjb200_stream_fold: summaries = one dict per shard with the fields of sjb200_stream_summary.  Returns
    (error, n_written, n, total_bytes, [per rank dict(kept, bytes_before, first_starts_document, rewrites=[(pos, val)])])"""
    from . import capi
    k = len(summaries)
    sums = (capi.StreamSummary * k)()
    for s, d in zip(sums, summaries):
        for name, _ in capi.StreamSummary._fields_:
            setattr(s, name, int(d.get(name, 0)))
    res = capi.StreamFoldResult()
    ranks = (capi.StreamRank * k)()
    _lib().sjb200_stream_fold(int(mode), k, int(final_state), int(flags_all), sums, C.byref(res), ranks)
    out = [{"kept": int(r.kept), "bytes_before": int(r.bytes_before), "first_starts_document": int(r.first_starts_document),
            "rewrites": [(int(r.rewrite_pos[j]), int(r.rewrite_val[j])) for j in range(r.nrewrites)]} for r in ranks]
    return int(res.error), int(res.n_written), int(res.n), int(res.total_bytes), out


def fold_delimited(mode, final_state, flags_all, summaries):
    """sjb200_delimited_fold: summaries = one dict per shard with the fields of sjb200_delimited_summary, `walk` and
    `walk_below` dicts with those of sjb200_stream_summary.  Returns (error, n_written, n, total_bytes, tail, [per rank
    dict(kept, filtered_before, bytes_before, first_starts_document)]); tail = 3 entries, each ("value", word) or
    ("filtered" | "scanned", rank, local position)"""
    from . import capi
    k = len(summaries)
    sums = (capi.DelimitedSummary * k)()
    for s, d in zip(sums, summaries):
        for name, _ in capi.DelimitedSummary._fields_:
            if name in ("walk", "walk_below"):
                for f, _ in capi.StreamSummary._fields_:
                    setattr(getattr(s, name), f, int(d.get(name, {}).get(f, 0)))
            else:
                setattr(s, name, int(d.get(name, 0)))
    res = capi.DelimitedFoldResult()
    ranks = (capi.DelimitedRank * k)()
    _lib().sjb200_delimited_fold(int(mode), k, int(final_state), int(flags_all), sums, C.byref(res), ranks)
    tail = [("value", int(res.tail_val[j])) if res.tail_rank[j] < 0 else
            ("filtered" if res.tail_filtered[j] else "scanned", int(res.tail_rank[j]), int(res.tail_pos[j])) for j in range(3)]
    out = [{"kept": int(r.kept), "filtered_before": int(r.filtered_before), "bytes_before": int(r.bytes_before),
            "first_starts_document": int(r.first_starts_document)} for r in ranks]
    return int(res.error), int(res.n_written), int(res.n), int(res.total_bytes), tail, out


def shard_cuts(buf, nshards):
    """cut a host buffer into nshards byte ranges at UTF-8 character boundaries"""
    L = _lib()
    a = np.ascontiguousarray(buf, dtype=np.uint8)
    cuts = [0]
    for k in range(1, nshards):
        cuts.append(int(L.sjb200_shard_cut(a.ctypes.data, len(a), (len(a) * k) // nshards)))
    cuts.append(len(a))
    return cuts


def shard_cuts_at_lines(buf, nshards, window=1 << 20):
    """the same, preferring cuts right after a raw line feed (a raw 0x0A cannot lie inside a JSON string, so for valid
    input every shard starts in state 0 and no rank ever scans twice)"""
    L = _lib()
    a = np.ascontiguousarray(buf, dtype=np.uint8)
    cuts = [0]
    for k in range(1, nshards):
        cuts.append(max(cuts[-1], int(L.sjb200_shard_cut_line(a.ctypes.data, len(a), (len(a) * k) // nshards, window))))
    cuts.append(len(a))
    return cuts


class Comm:
    """sjb200_comm: the per-rank object of the sharded scan with the exchange fused into the scan kernel
    (include/sjb200.h).  connect() maps the peers' exchange windows: pass `all_gather_bytes`, a callable that all-gathers
    a 64-byte uint8 array over the job's process group (torch.distributed over NCCL or gloo) -- the only collective of
    the path, once per job -- or, for ranks living in one process, connect_local()."""

    def __init__(self, parser, rank, world):
        from . import capi
        self._capi = capi
        self.parser, self.rank, self.world = parser, rank, world
        self._tokens_out = collections.deque()  # the outputs of the tokens passes in flight, oldest first
        self._grammar_out = collections.deque()  # ... and of the grammar passes
        self._pointer_out = collections.deque()  # ... and of the pointer passes
        self._h = C.c_void_p()
        rc = _lib().sjb200_comm_create(parser._ctx, rank, world, C.byref(self._h))
        if rc != 0:
            raise RuntimeError(f"sjb200_comm_create failed ({rc}): " + parser.last_cuda_error())

    def handle(self):
        h = np.zeros(self._capi.COMM_HANDLE_BYTES, dtype=np.uint8)
        rc = _lib().sjb200_comm_get_handle(self._h, h.ctypes.data)
        if rc != 0:
            raise RuntimeError("sjb200_comm_get_handle failed: " + self.parser.last_cuda_error())
        return h

    def connect(self, all_gather_bytes):
        if self.world == 1:
            return
        handles = np.ascontiguousarray(all_gather_bytes(self.handle()), dtype=np.uint8).reshape(self.world, self._capi.COMM_HANDLE_BYTES)
        rc = _lib().sjb200_comm_connect(self._h, handles.ctypes.data)
        if rc != 0:
            raise RuntimeError("sjb200_comm_connect failed: " + self.parser.last_cuda_error())

    @staticmethod
    def connect_local(comms):
        arr = (C.c_void_p * len(comms))(*[c._h for c in comms])
        for c in comms:
            rc = _lib().sjb200_comm_connect_local(c._h, arr)
            if rc != 0:
                raise RuntimeError("sjb200_comm_connect_local failed: " + c.parser.last_cuda_error())

    def enqueue(self, d_shard, d_idx, last_shard, stream=None):
        from .implementation import _stream_ptr
        return _lib().sjb200_stage1_sharded_enqueue(self._h, d_shard.data_ptr(), d_shard.numel(), int(last_shard), d_idx.data_ptr(), _stream_ptr(stream))

    def finish(self):
        res = self._capi.ShardedResult()
        rc = _lib().sjb200_stage1_sharded_finish(self._h, C.byref(res))
        return rc, res

    def scan(self, d_shard, d_idx, last_shard, stream=None):
        rc = self.enqueue(d_shard, d_idx, last_shard, stream)
        if rc != 0:
            return rc, None
        return self.finish()

    # minify and validate_utf8 passes go through the same window; every rank must enqueue the same sequence of kinds
    def minify_enqueue(self, d_shard, d_dst, stream=None):
        """d_dst: uint8 device tensor of at least d_shard.numel() bytes; the shard's kept bytes are d_dst[:count]"""
        from .implementation import _stream_ptr
        if d_dst.numel() * d_dst.element_size() < d_shard.numel():
            raise ValueError("d_dst needs len(shard) bytes")
        return _lib().sjb200_minify_sharded_enqueue(self._h, d_shard.data_ptr(), d_shard.numel(), d_dst.data_ptr(), _stream_ptr(stream))

    def minify_finish(self):
        """(error_code, ShardedResult): count kept bytes at offset base of the minified document of length total_count;
        UNCLOSED_STRING on every rank when the document ends inside a string"""
        res = self._capi.ShardedResult()
        rc = _lib().sjb200_minify_sharded_finish(self._h, C.byref(res))
        return rc, res

    def minify(self, d_shard, d_dst, stream=None):
        rc = self.minify_enqueue(d_shard, d_dst, stream)
        if rc != 0:
            return rc, None
        return self.minify_finish()

    def validate_utf8_enqueue(self, d_shard, stream=None):
        """cut the buffer at character boundaries (shard_cuts): then the AND of the shards' verdicts is the buffer's"""
        from .implementation import _stream_ptr
        return _lib().sjb200_validate_utf8_sharded_enqueue(self._h, d_shard.data_ptr(), d_shard.numel(), _stream_ptr(stream))

    def validate_utf8_finish(self):
        """(verdict, ShardedResult): 1 when the whole buffer is valid UTF-8, 0 when not, negative on a failure"""
        res = self._capi.ShardedResult()
        v = _lib().sjb200_validate_utf8_sharded_finish(self._h, C.byref(res))
        return v, res

    def validate_utf8(self, d_shard, stream=None):
        if self.validate_utf8_enqueue(d_shard, stream) != 0:
            return -1, None
        return self.validate_utf8_finish()

    # stage 1 of a whitespace-separated stream with the whole stream's finish() (modes REGULAR, STREAMING_PARTIAL,
    # STREAMING_FINAL); its passes share the window with the other kinds
    def stream_enqueue(self, d_shard, d_idx, last_shard, mode, stream=None):
        from .implementation import _stream_ptr
        return _lib().sjb200_stage1_sharded_stream_enqueue(self._h, d_shard.data_ptr(), d_shard.numel(), int(last_shard), int(mode), d_idx.data_ptr(),
                                                           _stream_ptr(stream))

    def stream_finish(self):
        """(error_code, ShardedStreamResult): the error code and n of stage1(whole stream, mode) on every rank; this
        shard's kept structurals d_idx[:kept] + bytes_before, total_bytes, first_starts_document"""
        res = self._capi.ShardedStreamResult()
        rc = _lib().sjb200_stage1_sharded_stream_finish(self._h, C.byref(res))
        return rc, res

    def scan_stream(self, d_shard, d_idx, last_shard, mode, stream=None):
        rc = self.stream_enqueue(d_shard, d_idx, last_shard, mode, stream)
        if rc != 0:
            return rc, None
        return self.stream_finish()

    # stage 1 of an RS-delimited (modes JSON_SEQUENCE_*) or comma-delimited (COMMA_DELIMITED_*) stream with the whole
    # stream's filter and finish(); its passes share the window with the other kinds
    def delimited_enqueue(self, d_shard, d_idx, last_shard, mode, stream=None):
        from .implementation import _stream_ptr
        return _lib().sjb200_stage1_sharded_delimited_enqueue(self._h, d_shard.data_ptr(), d_shard.numel(), int(last_shard), int(mode), d_idx.data_ptr(),
                                                              _stream_ptr(stream))

    def delimited_finish(self):
        """(error_code, ShardedDelimitedResult): the error code and n of stage1(whole stream, mode) on every rank; this
        shard's filtered entries d_idx[:filtered] (shard-relative), of which d_idx[:stream.kept] + stream.bytes_before are
        among the first n; tail = the whole call's words n, n+1, n+2"""
        res = self._capi.ShardedDelimitedResult()
        rc = _lib().sjb200_stage1_sharded_delimited_finish(self._h, C.byref(res))
        return rc, res

    def scan_delimited(self, d_shard, d_idx, last_shard, mode, stream=None):
        rc = self.delimited_enqueue(d_shard, d_idx, last_shard, mode, stream)
        if rc != 0:
            return rc, None
        return self.delimited_finish()

    # stage-2-lite over this shard's structurals; its passes share the window with the other kinds
    def tokens_enqueue(self, d_shard, d_idx, n, state_in, strbuf_capacity=None, stream=None):
        """(d_idx, n): this shard's structurals from a sharded stage-1 pass (count, or kept for a stream / delimited pass),
        state_in: that pass's folded state_in (it must be 0).  Allocates the outputs the way
        dom_parser_implementation.tokens_device does (string buffer: sjb200_string_buf_capacity(len(shard)) bytes by
        default) and keeps them until tokens_finish returns them."""
        import torch

        from .implementation import _stream_ptr
        n = int(n)
        cap = int(_lib().sjb200_string_buf_capacity(d_shard.numel())) if strbuf_capacity is None else int(strbuf_capacity)
        dev = d_shard.device
        d_type = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        d_payload = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        d_strbuf = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        rc = _lib().sjb200_tokens_sharded_enqueue(self._h, d_shard.data_ptr(), d_shard.numel(), int(state_in), d_idx.data_ptr(), n, d_type.data_ptr(),
                                                  d_payload.data_ptr(), d_strbuf.data_ptr() if cap else None, cap, _stream_ptr(stream))
        if rc == 0:
            self._tokens_out.append((d_type[:n], d_payload[:n], d_strbuf))
        return rc

    def tokens_finish(self):
        """(error_code, ShardedTokensResult, d_type uint8[n], d_payload int64[n] (bit pattern of the uint64), d_strbuf) of
        the oldest pass in flight.  Outputs are shard-relative: '"' payloads + string_base and 'd' payloads + bytes_before
        are the whole document's; d_strbuf[:string_bytes] is this rank's part of its string buffer."""
        res = self._capi.ShardedTokensResult()
        rc = _lib().sjb200_tokens_sharded_finish(self._h, C.byref(res))
        if rc == self._capi.UNEXPECTED_ERROR and "oldest pass in flight is of another kind" in self.parser.last_cuda_error():
            return rc, res, None, None, None  # (it stays in flight, and so do the outputs of the tokens passes)
        d_type, d_payload, d_strbuf = self._tokens_out.popleft() if self._tokens_out else (None, None, None)
        return rc, res, d_type, d_payload, d_strbuf

    def tokens(self, d_shard, d_idx, n, state_in, strbuf_capacity=None, stream=None):
        rc = self.tokens_enqueue(d_shard, d_idx, n, state_in, strbuf_capacity, stream)
        if rc != 0:
            return rc, None, None, None, None
        return self.tokens_finish()

    # stage-2 grammar over this shard's tokens; its passes share the window with the other kinds
    def document_errors_enqueue(self, d_type, d_payload, n, whole, table=None, max_depth=None, stream=None):
        """(d_type, d_payload, n): this rank's output of a sharded tokens pass.  whole = True: the ranks hold one document;
        else table is this rank's document table (a [ndocs, 2] array from document_table, or a device tensor of
        sjb200_doc_boundary; None or empty: no document starts here).  Allocates d_out (one 16-byte result per document
        that starts here) and keeps it until document_errors_finish returns it."""
        import torch

        from .implementation import _stream_ptr
        n = int(n)
        dev = d_type.device
        max_depth = self.parser.max_depth if max_depth is None else int(max_depth)
        d_docs, ndocs = None, 0
        if not whole and table is not None and len(table):
            if isinstance(table, torch.Tensor) and table.is_cuda:
                d_docs, ndocs = table, table.numel() * table.element_size() // 8
            else:
                arr = np.ascontiguousarray(np.asarray(table, dtype=np.int64).reshape(-1, 2).astype(np.uint32)).view(np.int32).reshape(-1)
                d_docs, ndocs = torch.from_numpy(arr.copy()).to(dev), len(arr) // 2
        nout = 1 if whole else ndocs
        d_out = torch.empty(max(nout, 1) * 2, dtype=torch.int64, device=dev)
        rc = _lib().sjb200_document_errors_sharded_enqueue(self._h, d_type.data_ptr() if n else None, d_payload.data_ptr() if n else None, n, int(bool(whole)),
                                                           d_docs.data_ptr() if ndocs else None, ndocs, max_depth, d_out.data_ptr(), _stream_ptr(stream))
        if rc == 0:
            self._grammar_out.append((d_out, d_docs, nout if (not whole or self.rank == 0) else 0))
        return rc

    def document_errors_finish(self):
        """(error_code, ShardedDocumentErrorsResult, errors int32[k], indexes uint64[k]) of the oldest pass in flight: the
        results of the k documents that start on this rank (whole mode: rank 0's one), global structural indexes"""
        res = self._capi.ShardedDocumentErrorsResult()
        rc = _lib().sjb200_document_errors_sharded_finish(self._h, C.byref(res))
        if rc == self._capi.UNEXPECTED_ERROR and "oldest pass in flight is of another kind" in self.parser.last_cuda_error():
            return rc, res, None, None
        d_out, _, k = self._grammar_out.popleft() if self._grammar_out else (None, None, 0)
        # d_out holds results on success, and after a bad table (every result UNEXPECTED_ERROR); else nothing was written
        written = rc == 0 or (rc == self._capi.UNEXPECTED_ERROR and res.ndocs > 0 and res.ndocs_in_error == res.ndocs
                              and res.first_error == self._capi.UNEXPECTED_ERROR)
        if d_out is None or not written or res.ndocs == 0:
            return rc, res, np.zeros(0, dtype=np.int32), np.zeros(0, dtype=np.uint64)
        out = d_out[: 2 * k].cpu().numpy().view(np.uint64).reshape(-1, 2)
        return rc, res, (out[:, 0] & 0xFFFFFFFF).astype(np.uint32).view(np.int32), out[:, 1].copy()

    def document_errors(self, d_type, d_payload, n, whole, table=None, max_depth=None, stream=None):
        rc = self.document_errors_enqueue(d_type, d_payload, n, whole, table, max_depth, stream)
        if rc != 0:
            return rc, None, None, None
        return self.document_errors_finish()

    # JSON Pointer lookup over this shard's tokens; its passes share the window with the other kinds
    def at_pointer_enqueue(self, pointers, d_type, d_payload, n, d_strbuf, string_bytes, whole, table=None, stream=None):
        """pointers: str or bytes, the same on every rank.  (d_type, d_payload, n, d_strbuf, string_bytes): this rank's
        output of a sharded tokens pass.  whole = True: the ranks hold one document; else table is this rank's document
        table (as for document_errors_enqueue).  Allocates d_out (npointers x the documents that start here, 16 bytes
        each) and keeps it until at_pointer_finish returns it."""
        import torch

        from .implementation import _stream_ptr
        n = int(n)
        dev = d_type.device
        d_docs, ndocs = self._device_table(table, whole, dev)
        enc = [p.encode() if isinstance(p, str) else bytes(p) for p in pointers]
        P = len(enc)
        bufs = [C.create_string_buffer(e, len(e)) for e in enc]
        ptrs = (C.c_void_p * max(P, 1))(*[C.addressof(b) for b in bufs])
        lens = (C.c_size_t * max(P, 1))(*[len(e) for e in enc])
        nout = 1 if whole else ndocs
        d_out = torch.empty(max(P * nout, 1) * 2, dtype=torch.int64, device=dev)
        rc = _lib().sjb200_at_pointer_sharded_enqueue(self._h, d_type.data_ptr() if n else None, d_payload.data_ptr() if n else None, n,
                                                      d_strbuf.data_ptr() if string_bytes else None, int(string_bytes), int(bool(whole)),
                                                      d_docs.data_ptr() if ndocs else None, ndocs, ptrs, lens, P, d_out.data_ptr(), _stream_ptr(stream))
        if rc == 0:
            self._pointer_out.append((d_out, d_docs, P, nout if (not whole or self.rank == 0) else 0))
        return rc

    def at_pointer_finish(self):
        """(error_code, ShardedPointerSummary, errors int32[P, k], indexes uint64[P, k]) of the oldest pass in flight: the
        results of every pointer in the k documents that start on this rank (whole mode: rank 0's one), global structural
        indexes (UINT64_MAX: none)"""
        res = self._capi.ShardedPointerSummary()
        rc = _lib().sjb200_at_pointer_sharded_finish(self._h, C.byref(res))
        if rc == self._capi.UNEXPECTED_ERROR and "oldest pass in flight is of another kind" in self.parser.last_cuda_error():
            return rc, res, None, None
        d_out, _, P, k = self._pointer_out.popleft() if self._pointer_out else (None, None, 0, 0)
        # d_out holds results on success, and after a bad table (every result UNEXPECTED_ERROR); else nothing was written
        written = rc == 0 or (rc == self._capi.UNEXPECTED_ERROR and "document table is not strictly ascending" in self.parser.last_cuda_error())
        if d_out is None or not written or res.ndocs == 0:
            return rc, res, np.zeros((P, 0), dtype=np.int32), np.zeros((P, 0), dtype=np.uint64)
        out = d_out[: 2 * P * k].cpu().numpy().view(np.uint64).reshape(P, k, 2)
        return rc, res, (out[:, :, 0] & 0xFFFFFFFF).astype(np.uint32).view(np.int32), out[:, :, 1].copy()

    def at_pointer(self, pointers, d_type, d_payload, n, d_strbuf, string_bytes, whole, table=None, stream=None):
        rc = self.at_pointer_enqueue(pointers, d_type, d_payload, n, d_strbuf, string_bytes, whole, table, stream)
        if rc != 0:
            return rc, None, None, None
        return self.at_pointer_finish()

    def _device_table(self, table, whole, dev):
        """(device tensor of sjb200_doc_boundary or None, entries) from a [ndocs, 2] array or a device tensor"""
        import torch
        if whole or table is None or not len(table):
            return None, 0
        if isinstance(table, torch.Tensor) and table.is_cuda:
            return table, table.numel() * table.element_size() // 8
        arr = np.ascontiguousarray(np.asarray(table, dtype=np.int64).reshape(-1, 2).astype(np.uint32)).view(np.int32).reshape(-1)
        return torch.from_numpy(arr.copy()).to(dev), len(arr) // 2

    def document_table(self, d_shard, d_idx, result, stream=None):
        """the document starts among this shard's kept structurals (result: a ShardedStreamResult, or the `stream` field of
        a ShardedDelimitedResult, over the filtered entries): (local structural
        index, shard-relative byte) pairs as an int64 [ndocs, 2] CPU array.  Not collective."""
        import torch

        from .implementation import _stream_ptr
        kept = int(result.kept)
        table = torch.empty(max(kept, 1) * 2, dtype=torch.int32, device=d_idx.device)
        nd = C.c_uint32(0)
        rc = _lib().sjb200_document_table_shard_dev(self.parser._ctx, d_shard.data_ptr(), d_idx.data_ptr(), kept, int(result.first_starts_document),
                                                    table.data_ptr(), max(kept, 1), C.byref(nd), _stream_ptr(stream))
        if rc != 0:
            raise RuntimeError(f"sjb200_document_table_shard_dev failed ({rc}): " + self.parser.last_cuda_error())
        return table[: 2 * nd.value].cpu().numpy().view(np.uint32).astype(np.int64).reshape(-1, 2)

    def close(self):
        if self._h:
            _lib().sjb200_comm_destroy(self._h)
            self._h = C.c_void_p()


def exchange(scan, rank, world, all_gather):
    """Run the protocol on one rank.
      scan(state_in) -> (ttable, count, flags)   scans this rank's shard (GPU: sjb200_stage1_shard_dev)
      all_gather(int64[4]) -> int64[world][4]     the collective (NCCL / gloo all_gather of 32 bytes per rank)
    Returns dict(state_in, base, count, flags, rescanned, ttables)."""
    tt, count, flags = scan(0)
    g = all_gather(np.array([tt, count, flags, 0], dtype=np.int64))
    states = fold_states([int(x) for x in g[:, 0]])
    rescanned = False
    if states[rank] != 0:
        tt2, count, flags = scan(states[rank])
        assert tt2 == tt, "a shard's transducer cannot depend on its incoming state"
        rescanned = True
    if any(s != 0 for s in states):  # somebody's count changed: publish the corrected counts
        g = all_gather(np.array([tt, count, flags, 0], dtype=np.int64))
    return {"state_in": states[rank], "base": int(g[:rank, 1].sum()), "count": int(count), "flags": int(np.bitwise_or.reduce(g[:, 2])),
            "rescanned": rescanned, "ttables": [int(x) for x in g[:, 0]], "total": int(g[:, 1].sum())}


def unpack_result(row):
    """int64[3] written by sjb200_stage1_shard_dev_enqueue -> (ttable, count, flags, state_out)"""
    count, st_tt, fl = int(row[0]), int(row[1]), int(row[2])
    return (st_tt >> 32) & 0xFFFFFFFF, count, fl & 0xFFFFFFFF, st_tt & 0xFFFFFFFF


def verify_speculation(gathered, rank):
    """gathered: int64[world][3] from the all-gather of one speculative pass.  Returns (ok_for_everyone, my_state_in, my_base)."""
    rows = [unpack_result(r) for r in gathered]
    states = fold_states([r[0] for r in rows])
    base = sum(r[1] for r in rows[:rank])
    return all(s == 0 for s in states), states[rank], base
