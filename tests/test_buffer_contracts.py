"""Every entry point reads only its input and writes only its outputs.

The parity tests give each input and output a fresh tensor of its own, so a read before or after the input, or a write
outside an output, changes nothing they look at.  Here the input is a view into one larger allocation whose other bytes
are hostile -- a pending escape, an open string, a partial UTF-8 character, an RS byte or a bracket before it; a quote, a
backslash, continuation bytes, digits, an atom's tail, control characters or an escape after it -- so that reading one
of them changes the result, and every output is a view into an allocation filled with a known pattern that must still
hold around it afterwards.  At least 4 KiB of slack on each side keeps every over-read or over-write of the kinds the
kernels could make (look-backs, vector probes, 16-byte copy-outs, TMA boxes) inside the test's own allocation: a
visible difference, never a fault.

The result on a document must not depend on its surroundings, so each call with hostile surroundings is compared with
the oracle on exactly the document's bytes and with the same call on space-padded surroundings.  Covers stage 1 (every
mode, the batch call over packed rows with packed index arrays, the shard call, the host-pointer call), minify,
validate_utf8, stage-2-lite, the document tables, and the sharded passes with every shard in its own hostile
allocation."""
import ctypes as C
import random
import threading

import numpy as np
import pytest
import torch

import delimited_shards as D
import oracle_lib as O
import simdjson_b200 as sj
import stream_shards as S
import token_fuzz as TF
from simdjson_b200 import corpus, sharding
from test_gpu_parity import TILE, _big_adversarial, _doc_starts, _raw_scan
from test_sharded_minify_utf8 import _kept
import test_sharded_delimited as TSD
import test_sharded_streams as TSS
import test_sharded_tokens as TST

pytestmark = pytest.mark.gpu

SLACK = 4096
PATTERN = 0xAB
OFFSETS = (0, 1, 3, 4, 8, 15, 16)
ELEM = 65536  # the largest scan element (kElemBytes)
# bytes before a document that change its result when read: escape carry, in-string state, pending UTF-8, RS / depth
PREFIXES = (b"\\", b"\\\\\\", b'"', b"\xf0\x9f\x98", b"\xe2", b"\xc3", b"\x1e", b"[")
# ... and after it: a quote, an escape, continuation bytes, invalid UTF-8, a longer number, an atom's tail, control chars
SUFFIXES = (b'"', b"\\", b"\x80\x80\x80", b"\xff", b"0123456789", b"e+7", b"rue", b"\x00\x01", b"\\u00")
LENGTHS = ([1, 2, 3, 4, 5, 15, 16, 17, 63, 64, 65, 127, 128, 129, 4095, 4096, 4097]
           + [4096 * k + r for k in (2, 7) for r in (0, 1, 127, 128, 4095)]
           + [TILE - 1, TILE + 1, ELEM - 1, ELEM + 1, 3 * ELEM + 4100, (1 << 20) + 13])
HEADS = (b"\x80", b'"', b"\\", b"7")
TAILS = (b"12", b"tru", b'"ab', b"\\", b"\xf0\x9f\x98", b"\xe2\x82\xac")


def L():
    return sj.lib()


def words_of(n):
    return int(L().sjb200_index_words(n))


# --------------------------------------------------------------------------- helpers
def _tile_ending(pat, n):
    """n bytes of pat repeated, ending with a whole pat (backslash runs of odd length, separated by 'x')"""
    unit = (b"x" + pat) if pat.strip(b"\\") == b"" else pat
    return (unit * (n // len(unit) + 2))[-n:] if n else b""


def _tile_starting(pat, n):
    return (pat * (n // len(pat) + 2))[:n]


def embed(b, offset, before=b" ", after=b" "):
    """(allocation, view): b at byte `offset` past a 16-byte boundary inside one CUDA allocation, after SLACK + offset
    bytes of `before` tiled up to it and followed by SLACK bytes of `after`"""
    b = bytes(b)
    pre = SLACK + offset
    host = np.frombuffer(_tile_ending(before, pre) + b + _tile_starting(after, SLACK), dtype=np.uint8).copy()
    base = torch.from_numpy(host).cuda()
    assert base.data_ptr() % 256 == 0
    return base, base[pre: pre + len(b)]


class Fenced:
    """an output of n elements of `dtype` at byte `align_offset` past a 16-byte boundary, inside an allocation whose other
    bytes hold PATTERN; check() asserts they still do"""

    def __init__(self, n, dtype, align_offset=0, device="cuda"):
        isz = torch.empty(0, dtype=dtype).element_size()
        assert align_offset % isz == 0
        self.start, self.nbytes = SLACK + align_offset, n * isz
        self.base = torch.full((self.start + self.nbytes + SLACK,), PATTERN, dtype=torch.uint8, device=device)
        self.view = self.base[self.start: self.start + self.nbytes].view(dtype)

    def ptr(self):
        return self.base.data_ptr() + self.start

    def check(self, what=None):
        a = self.base.cpu().numpy()
        outside = np.concatenate([a[: self.start], a[self.start + self.nbytes:]])
        bad = np.nonzero(outside != PATTERN)[0]
        # (offsets of the changed bytes: negative before the output, 0 and up past its end)
        assert len(bad) == 0, (what, "written outside the output", [int(k) - self.start for k in bad[:8]])

    def u32(self):
        return self.view.cpu().numpy().view(np.uint32)


def edge_doc(rng, n, k):
    """n bytes that start with a continuation byte, a quote, a backslash or a digit and end in a number, a truncated atom,
    an open string, a lone backslash, a partial or a complete UTF-8 character (k picks the pair)"""
    mid = bytearray(_big_adversarial(rng, max(n, 300))[:n] if n >= 64 else bytes(corpus.adversarial(rng, 200) * 4)[:n])
    mid = bytes(mid) + b" " * (n - len(mid))
    head, tail = HEADS[k % len(HEADS)], TAILS[(k // len(HEADS) + k) % len(TAILS)]
    if n >= len(head) + len(tail):
        mid = head + mid[len(head): n - len(tail)] + tail
    elif n:
        mid = tail[-n:]
    return mid


def stage1_dev(p, view, n, mode, idx_ptr):
    nn = C.c_uint32(O.N_SENTINEL)
    rc = L().sjb200_stage1_dev(p._ctx, view.data_ptr(), n, mode, idx_ptr, C.byref(nn), None)
    return rc, nn.value


def assert_same(got, want, ctx):
    assert got.err == want.err and got.n == want.n, (ctx, got.err, want.err, got.n, want.n)
    if want.wrote:
        a, b = got.words(), want.words()
        if not np.array_equal(a, b):
            k = int(np.argmax(a != b))
            raise AssertionError((ctx, "first differing word", k, a[max(0, k - 3): k + 4], b[max(0, k - 3): k + 4]))


def _surroundings(k):
    """the k-th (prefix, suffix) pair: every prefix and every suffix within max(len) consecutive k"""
    return PREFIXES[k % len(PREFIXES)], SUFFIXES[k % len(SUFFIXES)]


NPAIRS = max(len(PREFIXES), len(SUFFIXES))


@pytest.fixture(scope="module")
def port():
    return O.Port()


@pytest.fixture(scope="module")
def parser():
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(4 << 20)
    assert rc == sj.SUCCESS, sj.ERROR_NAMES.get(rc, rc)
    yield p
    p.close()


# --------------------------------------------------------------------------- a / c: input isolation and output fences
def test_stage1_dev_isolation_and_index_fence(parser, port):
    """sjb200_stage1_dev in all 7 modes up to 64 KiB, modes 0 and 2 above: the same result as the oracle on exactly the
    document whatever surrounds it, and no word outside sjb200_index_words(len) written"""
    rng = random.Random(corpus.SEED ^ 0xB0F)
    for li, n in enumerate(LENGTHS):
        doc = edge_doc(rng, n, li)
        modes = range(7) if n <= ELEM else (0, 2)
        want = {m: port.stage1(doc, m) for m in modes}
        for oi, off in enumerate(OFFSETS if n <= ELEM else (0, 1, 16)):
            pairs = [(b" ", b" ")] + [_surroundings(k) for k in range(NPAIRS)]
            for pi, (pre, suf) in enumerate(pairs):
                _, view = embed(doc, off, pre, suf)
                for m in modes:
                    if pi > 1 and n > ELEM and m != (pi % 2) * 2:
                        continue  # (big documents: each pair in one mode)
                    out = Fenced(words_of(n), torch.int32, 4 * ((oi + m) % 4))
                    rc, nn = stage1_dev(parser, view, n, m, out.ptr())
                    got = O.Stage1Result(rc, nn, out.u32())
                    assert_same(got, want[m], (n, off, pre, suf, m))
                    out.check((n, off, pre, suf, m))


def test_minify_and_utf8_dev_isolation_and_fence(parser, port):
    """sjb200_minify_dev with d_dst at every offset 0-15 (exactly len bytes, fenced) and sjb200_validate_utf8_dev"""
    rng = random.Random(corpus.SEED ^ 0xB1F)
    for li, n in enumerate(LENGTHS):
        doc = edge_doc(rng, n, li + 3)
        werr, wout = port.minify(doc)
        wutf8 = int(port.validate_utf8(doc))
        for oi, off in enumerate(OFFSETS):
            for k in range(-1, NPAIRS):
                pre, suf = (b" ", b" ") if k < 0 else _surroundings(k)
                _, view = embed(doc, off, pre, suf)
                dst = Fenced(n, torch.uint8, (oi * 5 + k) % 16)
                dl = C.c_size_t(0)
                rc = L().sjb200_minify_dev(parser._ctx, view.data_ptr(), n, dst.ptr(), C.byref(dl), None)
                assert rc == werr, (n, off, pre, suf, rc, werr)
                if werr == 0:
                    assert dl.value == len(wout) and bytes(dst.view[: dl.value].cpu().numpy()) == wout, (n, off, pre, suf)
                dst.check((n, off, pre, suf))
                assert L().sjb200_validate_utf8_dev(parser._ctx, view.data_ptr(), n, None) == wutf8, (n, off, pre, suf)


def _scan_shard(port, doc, state_in):
    Lp = port.L
    Lp.sjo_scan_shard.restype = C.c_uint64
    Lp.sjo_scan_shard.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    a = np.frombuffer(bytes(doc), dtype=np.uint8)
    idx = np.zeros(len(a) + 4, dtype=np.uint32)
    so = C.c_uint32(0)
    k = Lp.sjo_scan_shard(a.ctypes.data, len(a), state_in, idx.ctypes.data, C.byref(so))
    return idx[: int(k)], int(so.value)


def test_shard_dev_isolation_and_fence(parser, port):
    """sjb200_stage1_shard_dev in every incoming state 0..7 against the oracle's scan of exactly the shard"""
    rng = random.Random(corpus.SEED ^ 0xB2F)
    for li, n in enumerate([x for x in LENGTHS if x <= ELEM + 1]):
        doc = edge_doc(rng, n, li + 5)
        wants = [_scan_shard(port, doc, s) for s in range(8)]
        for j, (off, k) in enumerate((off, k) for off in OFFSETS for k in range(NPAIRS)):
            # every prefix and every suffix at each (length, offset); every incoming state at each offset
            state_in = (k + off) % 8
            want, wstate = wants[state_in]
            pre, suf = _surroundings(k)
            _, view = embed(doc, off, pre, suf)
            out = Fenced(words_of(n), torch.int32, 4 * (j % 4))
            res = sj.capi.ShardResult()
            rc = L().sjb200_stage1_shard_dev(parser._ctx, view.data_ptr(), n, state_in, j % 2, out.ptr(), C.byref(res), None)
            ctx = (n, off, pre, suf, state_in)
            assert rc == 0 and res.count == len(want) and res.state_out == wstate & 7, (ctx, res.count, len(want))
            assert np.array_equal(out.u32()[: res.count], want), ctx
            assert bool(res.flags & 1) == (not port.validate_utf8(doc)), ctx
            out.check(ctx)


def _token_docs(rng):
    """documents stage 1 accepts whose first and last bytes belong to a number, an atom, a string or an escape"""
    docs = [b"[1,23", b"7", b"-1.5e+1", b"[true,fals", b"[null,tru", b'"\\\\"', b'["a\\u00e9","\\ud83d\\ude00"', b'"\\u00e9"', b'"x\\""',
            b'{"k":123456789012345678', b"[1.0e", b'["\xf0\x9f\x98\x80"', b"[-0,", b'""']
    for k in range(24):
        parts = []
        for _ in range(rng.randrange(1, 400)):
            if rng.random() < 0.5:
                parts.append(b'"' + TF.string_body(rng)[0] + b'"')
            else:
                tok = TF.scalar_token(rng)
                if b'"' not in tok and b"\\" not in tok:
                    parts.append(tok)
        d = b"[" + b",".join(parts)
        if k % 3 == 0:
            d += b"]"
        docs.append(d)
    docs.append(b'["' + TF.long_body(rng, 70000, 0.3) + b'",' + b"12" * 3)
    return docs


def _tokens_call(p, view, n_bytes, d_idx_ptr, n, cap, ty_off=0, sb_off=0):
    ty = Fenced(n, torch.uint8, ty_off)
    pl = Fenced(n, torch.int64, 8 * (ty_off % 2))
    sb = Fenced(cap, torch.uint8, sb_off)
    res = sj.capi.TokensResult()
    L().sjb200_tokens_dev(p._ctx, view.data_ptr(), n_bytes, d_idx_ptr, n, ty.ptr(), pl.ptr(), sb.ptr() if cap else None, cap, C.byref(res), None)
    torch.cuda.synchronize()
    return res, ty, pl, sb


def _same_tokens(res, ty, pl, sb, want, ctx, capacity_error=False):
    err, types, pay, sbytes, sl, ns, fe = want
    assert res.error == err and res.string_bytes == sl and res.n_strings == ns and res.first_error_index == fe, (ctx, res.error, err)
    assert bytes(ty.view.cpu().numpy()) == bytes(types), (ctx, "types")
    assert np.array_equal(pl.view.cpu().numpy().view(np.uint64), pay), (ctx, "payloads")
    if not capacity_error:
        assert bytes(sb.view[: sl].cpu().numpy()) == bytes(sbytes), (ctx, "string_buf")
    ty.check((ctx, "types")); pl.check((ctx, "payloads")); sb.check((ctx, "string_buf"))


def test_tokens_dev_isolation_and_fences(parser, port):
    """sjb200_tokens_dev on documents whose last token ends on the last byte, followed by bytes that would extend it;
    d_type / d_payload exactly n entries, d_strbuf at offsets 0-15, all fenced; capacity exactly string_bytes (SUCCESS),
    one byte less (CAPACITY: nothing written to d_strbuf, payloads the oracle's lengths), and n = 0"""
    rng = random.Random(corpus.SEED ^ 0xB3F)
    for di, doc in enumerate(_token_docs(rng)):
        r = port.stage1(doc)
        assert r.err == 0, doc[:40]
        d_idx = torch.from_numpy(np.ascontiguousarray(r.idx[: r.n + 3]).view(np.int32)).cuda()
        full_cap = int(L().sjb200_string_buf_capacity(len(doc)))
        want = port.tokens(doc, r.idx, r.n, strbuf_cap=full_cap)
        sl = want[4]
        for k in range(NPAIRS if di < 16 else 2):
            pre, suf = _surroundings(k + di)
            off = OFFSETS[(k + di) % len(OFFSETS)]
            _, view = embed(doc, off, pre, suf)
            ctx = (doc[:40], off, pre, suf)
            res, ty, pl, sb = _tokens_call(parser, view, len(doc), d_idx.data_ptr(), r.n, full_cap, k % 16, (k * 7) % 16)
            _same_tokens(res, ty, pl, sb, want, ctx)
            if k < 2 and want[0] == 0:
                res, ty, pl, sb = _tokens_call(parser, view, len(doc), d_idx.data_ptr(), r.n, int(sl), 0, (k * 5 + di) % 16)
                _same_tokens(res, ty, pl, sb, want, (ctx, "exact capacity"))
                if sl > 0:
                    wantc = port.tokens(doc, r.idx, r.n, strbuf_cap=int(sl) - 1)
                    assert wantc[0] == sj.CAPACITY
                    res, ty, pl, sb = _tokens_call(parser, view, len(doc), d_idx.data_ptr(), r.n, int(sl) - 1, 0, (k * 3 + di) % 16)
                    assert bytes(sb.view.cpu().numpy()) == bytes([PATTERN]) * (int(sl) - 1), (ctx, "CAPACITY wrote to d_strbuf")
                    _same_tokens(res, ty, pl, sb, wantc, (ctx, "capacity - 1"), capacity_error=True)
        res, ty, pl, sb = _tokens_call(parser, view, len(doc), d_idx.data_ptr(), 0, 16, 0, 3)
        assert res.error == 0 and res.n_strings == 0 and res.string_bytes == 0 and res.first_error_index == 0xFFFFFFFF
        ty.check("n=0"); pl.check("n=0"); sb.check("n=0")
        assert bytes(sb.view.cpu().numpy()) == bytes([PATTERN]) * 16


def _table(p, view, d_idx_ptr, n, capacity, first_starts=None, off=0):
    t = Fenced(2 * capacity, torch.int32, off)
    nd = C.c_uint32(0xDEAD)
    if first_starts is None:
        rc = L().sjb200_document_table_dev(p._ctx, view.data_ptr(), d_idx_ptr, n, t.ptr(), capacity, C.byref(nd), None)
    else:
        rc = L().sjb200_document_table_shard_dev(p._ctx, view.data_ptr(), d_idx_ptr, n, first_starts, t.ptr(), capacity, C.byref(nd), None)
    torch.cuda.synchronize()
    return rc, nd.value, t


def test_document_tables_isolation_and_capacity(parser, port):
    """sjb200_document_table_dev / _shard_dev with capacity 0, 1, ndocs - 1, ndocs, ndocs + 1: *ndocs_out is the true
    count, the first min(capacity, ndocs) entries are right, nothing past capacity is written"""
    rng = random.Random(corpus.SEED ^ 0xB4F)
    docs = [bytes(corpus.multi_document(rng)) for _ in range(12)] + [bytes(corpus.ndjson_rows(300000))[:-77], b"1 2 3", b"[1] [2",
                                                                        bytes(corpus.tile_documents([b'{"k":[1,2]}', b"7", b'"s"'], 70000))]
    for di, doc in enumerate(docs):
        r = port.stage1(doc, 2)
        if r.err != 0 or r.n == 0:
            continue
        a = np.frombuffer(doc, dtype=np.uint8)
        idx = r.idx[: r.n].astype(np.int64)
        starts = _doc_starts(a, idx)
        nd = len(starts)
        d_idx = torch.from_numpy(np.ascontiguousarray(r.idx[: r.n + 3]).view(np.int32)).cuda()
        for ci, cap in enumerate(sorted({0, 1, max(nd - 1, 0), nd, nd + 1})):
            pre, suf = _surroundings(di + ci)
            _, view = embed(doc, OFFSETS[(di + ci) % len(OFFSETS)], pre, suf)
            for shard in (None, 1, 0):
                rc, got_nd, t = _table(parser, view, d_idx.data_ptr(), r.n, cap, shard, 4 * ci % 16)
                wst = starts if shard != 0 else starts[1:]
                ctx = (di, cap, shard, pre, suf)
                assert rc == 0 and got_nd == len(wst), (ctx, got_nd, len(wst))
                k = min(cap, len(wst))
                tab = t.u32().reshape(-1, 2)[:k] if cap else np.zeros((0, 2), np.uint32)
                assert np.array_equal(tab[:, 0], wst[:k]) and np.array_equal(tab[:, 1], idx[wst[:k]]), ctx
                t.check(ctx)


# --------------------------------------------------------------------------- b: packed batch
def _packed_docs(rng):
    rows = [r + b"\n" for r in bytes(corpus.ndjson_rows(200000)).split(b"\n") if r][:60]
    docs = rows[:]
    docs += [bytes(corpus.adversarial(rng)) for _ in range(40)]
    docs += [b'{"a": "x\\', b'{"a": "open string', b"[1, \"\xe2", b'{"k": "\xf0\x9f', b"", b"", b'"\\\\\\', b"12", b"tru", b"\x1e[1]\x1e"]
    docs += [_big_adversarial(rng, n) for n in (4096, 4097, TILE + 7, 2 * ELEM + 1)]
    docs += [b""] * 3
    rng.shuffle(docs)
    # every other document is followed by an empty one, whose index array nothing may write: a document that writes past
    # its own sjb200_index_words(len) words lands there whatever the order of the writes (the others keep non-empty
    # neighbours, as real rows have)
    out = []
    for k, b in enumerate(docs):
        out.append(b)
        if k % 2 == 0 and b:
            out.append(b"")
    return out


@pytest.mark.parametrize("pdl", [0, 1])
def test_batch_of_packed_rows(parser, port, pdl):
    """sjb200_stage1_dev_batch on consecutive, gapless views of one allocation (NDJSON rows in HBM, whose neighbours end in
    a backslash, inside a string or on a UTF-8 lead byte) with consecutive index arrays of exactly sjb200_index_words
    words each: every document equals the oracle and its own (fenced) sjb200_stage1_dev call, the index array of an empty
    document is not touched (a neighbour writing past its own words would land there), the fence after the last holds"""
    rng = random.Random(corpus.SEED ^ 0xB5F ^ pdl)
    docs = _packed_docs(rng)
    parser.set_option("pdl", pdl)
    try:
        for mode in range(7):
            blob = b"".join(docs)
            _, whole = embed(blob, 3 + mode, b"\\", b'"')
            words = [words_of(len(b)) for b in docs]
            out = Fenced(sum(words), torch.int32, 4 * (mode % 4))
            d_bufs, d_idxs, pos, w = [], [], 0, 0
            for b, k in zip(docs, words):
                d_bufs.append(whole[pos: pos + len(b)])
                d_idxs.append(out.view[w: w + k])
                pos += len(b)
                w += k
            res = parser.stage1_device_batch(d_bufs, d_idxs, mode)
            torch.cuda.synchronize()
            out.check(("batch", mode, pdl))
            allw = out.u32()
            w = 0
            for i, (b, (err, n)) in enumerate(zip(docs, res)):
                want = port.stage1(b, mode)
                got = O.Stage1Result(err, n if want.wrote else O.N_SENTINEL, allw[w: w + words[i]])
                if not want.wrote:
                    assert err == want.err, (i, mode, err, want.err)
                else:
                    assert_same(got, want, (i, len(b), mode, pdl))
                if len(b) == 0:
                    assert np.all(allw[w: w + words[i]] == 0xABABABAB), (i, mode, "an empty document's index array was written")
                if len(b):
                    own = Fenced(words[i], torch.int32, 4 * (i % 4))
                    rc, nn = stage1_dev(parser, d_bufs[i], len(b), mode, own.ptr())
                    assert rc == err and (not want.wrote or (nn == n and np.array_equal(own.u32()[: n + 3], allw[w: w + n + 3]))), (i, mode)
                    own.check(("own call", i, mode))
                w += words[i]
    finally:
        parser.set_option("pdl", 1)


# --------------------------------------------------------------------------- c: host-pointer calls
def test_host_pointer_calls_fenced(port):
    """sjb200_stage1 with idx_out exactly sjb200_index_words(capacity) words inside a fenced numpy array, pageable and
    page-locked, indexes copied back or stored by the kernel (zero_copy_out 0 / 1); sjb200_minify with dst exactly len
    bytes"""
    rng = random.Random(corpus.SEED ^ 0xB6F)
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(3 << 20)
    assert rc == sj.SUCCESS
    try:
        for li, n in enumerate((1, 129, 4097, TILE + 1, (1 << 20) + 13, 3 << 20)):
            doc = np.frombuffer(edge_doc(rng, n, li), dtype=np.uint8)
            cap = p.capacity()
            for mode in (0, 2, 4):
                want = port.stage1(doc, mode)
                for zc in (0, 1):
                    for pinned in (0, 1):
                        p.set_option("zero_copy_out", zc)
                        wds = words_of(cap)
                        host = np.full(SLACK + wds + SLACK, 0xABABABAB, dtype=np.uint32)
                        if pinned:
                            assert L().sjb200_pin_host_memory(p._ctx, host.ctypes.data, host.nbytes) == 0
                        try:
                            nn = C.c_uint32(O.N_SENTINEL)
                            rcs = L().sjb200_stage1(p._ctx, doc.ctypes.data, n, mode, host[SLACK:].ctypes.data, C.byref(nn))
                        finally:
                            if pinned:
                                L().sjb200_unpin_host_memory(p._ctx, host.ctypes.data)
                        ctx = (n, mode, zc, pinned)
                        assert_same(O.Stage1Result(rcs, nn.value, host[SLACK: SLACK + wds]), want, ctx)
                        assert np.all(host[:SLACK] == 0xABABABAB) and np.all(host[SLACK + wds:] == 0xABABABAB), ctx
            werr, wout = port.minify(doc)
            dst = np.full(SLACK + n + SLACK, PATTERN, dtype=np.uint8)
            dl = C.c_size_t(0)
            assert L().sjb200_minify(p._ctx, doc.ctypes.data, n, dst[SLACK:].ctypes.data, C.byref(dl)) == werr
            if werr == 0:
                assert bytes(dst[SLACK: SLACK + dl.value]) == wout
            assert np.all(dst[:SLACK] == PATTERN) and np.all(dst[SLACK + n:] == PATTERN), n
    finally:
        p.set_option("zero_copy_out", 0)
        p.close()


# --------------------------------------------------------------------------- d: index words past n
def test_index_words_past_n_are_not_read(parser, port):
    """sjb200_tokens_dev and the document tables with n below the stage-1 count (what the sharded stream and delimited
    passes do with `kept`), d_idx[n:] overwritten with hostile words: the outputs are those of the first n structurals"""
    rng = random.Random(corpus.SEED ^ 0xB7F)
    rows, _ = TST._array_doc(rng, 400)
    long_str = b'["' + TF.long_body(rng, 50000, 0.2) + b'", 1, "ab"]'
    for doc in (rows, long_str):
        a = np.frombuffer(doc, dtype=np.uint8)
        r = port.stage1(a)
        assert r.err == 0
        full_cap = int(L().sjb200_string_buf_capacity(len(doc)))
        quote = int(np.nonzero(a == ord('"'))[0][-1])
        ns = [1, 255, 256, 257] if doc is rows else [1, 2]  # (long_str: n = 2 ends on the open quote of a 50 KB string)
        _, view = embed(doc, 1, b"\\", b'"')
        d_full = torch.from_numpy(r.idx[: r.n + 3].view(np.int32).copy()).cuda()
        fres, fty, fpl, fsb = _tokens_call(parser, view, len(doc), d_full.data_ptr(), r.n, full_cap)
        for n in ns:
            want = port.tokens(a, r.idx, n, strbuf_cap=full_cap)
            for junk in (0, 0xFFFFFFFF, len(doc), quote):
                hi = r.idx[: r.n + 3].copy()
                hi[n:] = junk
                d_idx = torch.from_numpy(hi.view(np.int32)).cuda()
                res, ty, pl, sb = _tokens_call(parser, view, len(doc), d_idx.data_ptr(), n, full_cap, n % 16, junk % 16)
                _same_tokens(res, ty, pl, sb, want, (len(doc), n, junk))
                assert bytes(ty.view.cpu().numpy()) == bytes(fty.view[:n].cpu().numpy())
                assert bytes(sb.view[: res.string_bytes].cpu().numpy()) == bytes(fsb.view[: res.string_bytes].cpu().numpy())
                rc2 = port.stage1(a, 2)
                starts = _doc_starts(a, rc2.idx[:n].astype(np.int64))
                rc, nd, t = _table(parser, view, d_idx.data_ptr(), n, n + 1)
                assert rc == 0 and nd == len(starts) and np.array_equal(t.u32().reshape(-1, 2)[:nd, 0], starts), (n, junk)
                t.check((n, junk))


# --------------------------------------------------------------------------- e: sharded passes, each shard in its own hostile allocation
def _run_ranks_embedded(shards, body, salt=0, device=0):
    """like test_sharded_minify_utf8._run_ranks, but rank r's shard is embed()ded with a hostile prefix and suffix (on
    several GPUs the bytes before a shard are another allocation or unmapped memory)"""
    world = len(shards)
    impl = sj.get_active_implementation(device)
    parsers, comms = [], []
    for r in range(world):
        rc, p = impl.create_dom_parser_implementation(max(len(shards[r]), 64))
        assert rc == sj.SUCCESS
        parsers.append(p)
        comms.append(sharding.Comm(p, r, world))
    sharding.Comm.connect_local(comms)
    out = [None] * world

    def work(r):
        try:
            torch.cuda.set_device(device)
            pre, suf = _surroundings(r + salt)
            keep, d = embed(bytes(np.asarray(shards[r], dtype=np.uint8)), OFFSETS[(r + salt) % len(OFFSETS)], pre, suf)
            out[r] = body(r, comms[r], parsers[r], d, torch.cuda.Stream())
            del keep
        except Exception as e:  # noqa: BLE001
            out[r] = e

    th = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    [t.start() for t in th]
    [t.join(timeout=300) for t in th]
    assert not any(t.is_alive() for t in th), "a rank did not finish"
    for c in comms:
        c.close()
    for p in parsers:
        p.close()
    for o in out:
        if isinstance(o, Exception) or o is None:
            raise AssertionError(o)
    return out


def _fenced_stage1_body(r, comm, p, d, stream):
    out = Fenced(words_of(d.numel()), torch.int32, 4 * (r % 4))
    rc, x = comm.scan(d, out.view, r == comm.world - 1, stream)
    torch.cuda.synchronize()
    out.check(("sharded stage 1", r))
    return rc, int(x.count), int(x.base), out.u32()[: int(x.count)].astype(np.int64)


def _fenced_minify_body(r, comm, p, d, stream):
    dst = Fenced(d.numel(), torch.uint8, (5 * r + 3) % 16)
    rc, x = comm.minify(d, dst.view, stream)
    torch.cuda.synchronize()
    dst.check(("sharded minify", r))
    return rc, int(x.count), int(x.base), bytes(dst.view[: int(x.count)].cpu().numpy())


def _validate_body(r, comm, p, d, stream):
    v, _ = comm.validate_utf8(d, stream)
    torch.cuda.synchronize()
    return v


def test_sharded_passes_in_hostile_allocations(port):
    """sjb200_stage1_sharded (byte and line cuts), minify and validate_utf8 with 2 and 4 ranks, each shard embedded with a
    hostile prefix and suffix, every rank's output fenced: the gathered outputs equal one pass over the whole buffer"""
    rng = random.Random(corpus.SEED ^ 0xB8F)
    docs = [corpus.ndjson_rows(1 << 20), np.frombuffer(_big_adversarial(rng, 5 * TILE + 777), dtype=np.uint8).copy()]
    for di, doc in enumerate(docs):
        want, _ = _raw_scan(port, doc)
        werr, wmin = _kept(port, doc)
        wutf8 = int(port.validate_utf8(doc))
        for world in (2, 4):
            for how, cuts in (("bytes", sharding.shard_cuts(doc, world)), ("lines", sharding.shard_cuts_at_lines(doc, world))):
                if any(cuts[k + 1] <= cuts[k] for k in range(world)):
                    continue
                shards = [doc[cuts[r]: cuts[r + 1]] for r in range(world)]
                outs = _run_ranks_embedded(shards, _fenced_stage1_body, salt=di + world)
                got = np.concatenate([o[3] + cuts[r] for r, o in enumerate(outs)])
                assert all(o[0] == 0 for o in outs) and np.array_equal(got, want), (di, world, how)
                outs = _run_ranks_embedded(shards, _fenced_minify_body, salt=di + world + 1)
                assert all(o[0] == werr for o in outs) and b"".join(o[3] for o in outs) == wmin, (di, world, how)
                outs = _run_ranks_embedded(shards, _validate_body, salt=di + world + 2)
                assert all(v == wutf8 for v in outs), (di, world, how)


def _fenced_stream_body(world):
    """test_sharded_streams._stream_body with every mode's index buffer fenced: the last rank's sentinels, the streaming
    rewrites placed by the cross-rank fold and the document table all stay inside sjb200_index_words(len) words"""
    def body(r, comm, p, d, stream):
        last = r == world - 1
        fences = [Fenced(words_of(d.numel()), torch.int32, 4 * ((r + k) % 4)) for k in range(len(TSS.MODES))]
        for mode, f in zip(TSS.MODES, fences):
            assert comm.stream_enqueue(d, f.view, last, mode, stream) == 0
        out = []
        for mode, f in zip(TSS.MODES, fences):
            rc, x = comm.stream_finish()
            torch.cuda.synchronize()
            count = int(x.shard.count)
            words = f.view[: count + (3 if last else 0)].cpu().numpy().view(np.uint32).copy()
            table = comm.document_table(d, f.view, x, stream) if mode == O.STREAMING_FINAL else None
            torch.cuda.synchronize()
            f.check(("sharded stream", world, r, mode))
            out.append(dict(err=rc, n=int(x.n), kept=int(x.kept), bytes_before=int(x.bytes_before), total_bytes=int(x.total_bytes),
                            first_starts_document=int(x.first_starts_document), count=count, words=words, table=table,
                            rescanned=int(x.shard.rescanned)))
        return out
    return body


def _fenced_delimited_body(world):
    """test_sharded_delimited._delimited_body with every mode's index buffer fenced: the filter's compaction of the kept
    entries and the tail words stay inside sjb200_index_words(len) words"""
    def body(r, comm, p, d, stream):
        last = r == world - 1
        fences = [Fenced(words_of(d.numel()), torch.int32, 4 * ((r + k) % 4)) for k in range(len(D.MODES))]
        for mode, f in zip(D.MODES, fences):
            assert comm.delimited_enqueue(d, f.view, last, mode, stream) == 0
        out = []
        for mode, f in zip(D.MODES, fences):
            rc, x = comm.delimited_finish()
            torch.cuda.synchronize()
            g = TSD._result(rc, x, f.view)
            g["table"] = comm.document_table(d, f.view, x.stream, stream)
            torch.cuda.synchronize()
            f.check(("sharded delimited", world, r, mode))
            out.append(g)
        return out
    return body


def test_sharded_stream_and_delimited_passes_in_hostile_allocations():
    """the stream pass (modes 0-2) and the delimited pass (modes 3-6), shards embedded, every rank's index buffers fenced,
    against stage1(whole buffer)"""
    oracle = S.Oracle()
    rng = random.Random(corpus.SEED ^ 0xB9F)
    rows = [r for r in bytes(corpus.ndjson_rows(600000)).split(b"\n") if r]
    bufs = [("ndjson", b"\n".join(rows) + b"\n"), ("ndjson_cut", (b"\n".join(rows))[:-97])]
    for name, buf in bufs:
        for world in (2, 4):
            for cuts in S.cut_sets(rng, buf, world, 1) + [sharding.shard_cuts_at_lines(np.frombuffer(buf, dtype=np.uint8), world, window=len(buf) // (2 * world))]:
                if any(cuts[k + 1] <= cuts[k] for k in range(world)) or oracle.shards(buf, cuts, O.STREAMING_FINAL) is None:
                    continue
                outs = _run_ranks_embedded([np.frombuffer(buf[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(world)], _fenced_stream_body(world), salt=world)
                TSS._check_pass(oracle, buf, cuts, outs)
    dbufs = [("rs", b"".join(b"\x1e" + r + b"\n" for r in rows[:800])), ("comma", b",\n".join(rows[:800])[:-51])]
    for name, buf in dbufs:
        for world in (2, 4):
            for cuts in [sharding.shard_cuts(np.frombuffer(buf, dtype=np.uint8), world),
                         sharding.shard_cuts_at_lines(np.frombuffer(buf, dtype=np.uint8), world, window=len(buf) // (2 * world))]:
                if any(cuts[k + 1] <= cuts[k] for k in range(world)) or oracle.shards(buf, cuts, O.JSON_SEQUENCE_FINAL) is None:
                    continue
                outs = _run_ranks_embedded([np.frombuffer(buf[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(world)], _fenced_delimited_body(world), salt=world + 1)
                TSD._check_pass(oracle, buf, cuts, outs)


def test_sharded_tokens_in_hostile_allocations(port):
    """sjb200_stage1_sharded then sjb200_tokens_sharded at line cuts, shards embedded: the gathered outputs equal the
    oracle's tokens of the whole document"""
    rng = random.Random(corpus.SEED ^ 0xBAF)
    doc, _ = TST._array_doc(rng, 3000)
    a = np.frombuffer(doc, dtype=np.uint8)
    w = port.stage1(a)
    assert w.err == 0
    want = port.tokens(a, w.idx, w.n, strbuf_cap=int(L().sjb200_string_buf_capacity(len(doc))))
    for world in (2, 4):
        cuts = sharding.shard_cuts_at_lines(a, world, window=len(a) // (2 * world))
        outs = _run_ranks_embedded([a[cuts[r]: cuts[r + 1]] for r in range(world)], TST._stage1_body(), salt=world)
        TST._check(outs, want, ("tokens", world))
