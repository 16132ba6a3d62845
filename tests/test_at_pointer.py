"""sjb200_at_pointer_dev on the H100 against the JSON Pointer oracle (sjo_at_pointer, pinned to the reference's
dom::element::at_pointer by tests/test_pointer_oracle.py): every pointer of tests/pointer_cases.py in every document,
NDJSON streams with the device document table, documents walked by a warp and by a CTA, bad tables, limits and a fenced
output buffer."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

import oracle_lib as O
import pointer_oracle as PO
import pointer_cases as PC
import simdjson_b200 as sj
from simdjson_b200 import capi, corpus

pytestmark = pytest.mark.gpu

CTA_MIN = 4096  # SJB200_POINTER_CTA_MIN: documents above it are walked by a CTA


@pytest.fixture(scope="module")
def parser():
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(64 << 20)
    assert rc == sj.SUCCESS
    yield p
    p.close()


def device_tokens(p, doc, mode=sj.REGULAR):
    d = torch.frombuffer(bytearray(doc), dtype=torch.uint8).cuda()
    assert p.stage1_device(d, mode) == sj.SUCCESS
    res, d_type, d_payload, d_strbuf = p.tokens_device(d)
    return d, res, d_type, d_payload, d_strbuf


def device_table(p, d, n):
    table = torch.zeros(2 * (n + 8), dtype=torch.int32, device="cuda")
    nd = C.c_uint32(0)
    assert sj.lib().sjb200_document_table_dev(p._ctx, d.data_ptr(), p.device_index_buffer().data_ptr(), n, table.data_ptr(), n + 8, C.byref(nd), None) == 0
    return table, nd.value


def check(p, doc, pointers, stream=False):
    port = PO.Pointers()
    d, res, d_type, d_payload, d_strbuf = device_tokens(p, doc)
    n = p.n_structural_indexes
    if stream:
        table, nd = device_table(p, d, n)
        starts = table[: 2 * nd].view(-1, 2)[:, 0].cpu().numpy().tolist()
        r, _tw, _s, want_err, want_idx = port.table(doc, pointers, starts=starts)
        assert starts == PO.document_starts(doc, r.idx, r.n)
        err, idx = p.at_pointer_device(pointers, d_type, d_payload, d_strbuf, res.string_bytes, d_docs=table, ndocs=nd)
    else:
        _r, _tw, _s, want_err, want_idx = port.table(doc, pointers)
        err, idx = p.at_pointer_device(pointers, d_type, d_payload, d_strbuf, res.string_bytes)
    err = err.cpu().numpy()
    idx = idx.cpu().numpy().view(np.uint32)
    bad = np.argwhere((err != want_err) | (idx != want_idx))
    assert len(bad) == 0, [(pointers[i], j, int(err[i, j]), int(want_err[i, j]), int(idx[i, j]), int(want_idx[i, j])) for i, j in bad[:8]]
    return err, idx


def test_corpus_documents(parser):
    for name, doc, pointers in PC.corpus_cases(full=True):
        check(parser, doc, pointers)


def test_ndjson_rows(parser):
    tw_ptrs = ["/id", "/user/id", "/user/screen_name", "/entities/hashtags/0/text", "/retweeted_status/user/id", "/text", "/x", "", "/0"]
    err, _ = check(parser, PC.stream_of(PC.twitter_rows()), tw_ptrs, stream=True)
    assert (err[0] == 0).all() and err.shape == (len(tw_ptrs), 100)
    am_ptrs = [f"/{i}" for i in range(10)] + ["/-", "/a", "/01", ""]
    check(parser, PC.stream_of(PC.amazon_rows(794)), am_ptrs, stream=True)
    # a stream of every small and bad document, and concatenated (whitespace-separated) documents
    docs = [d for d, _ in PC.SMALL] + PC.BAD + PC.random_docs(6, 11)
    ptrs = sorted({q for _, ps in PC.SMALL for q in ps} | {"/0/0", "/1", "/a"})
    check(parser, b"\n".join(docs), ptrs, stream=True)
    check(parser, b" ".join(docs), ptrs, stream=True)


def long_array(n_elems):
    return json.dumps([{"i": i, "v": [i, str(i)]} if i % 3 else i for i in range(n_elems)]).encode()


def test_documents_over_the_warp_limit(parser):
    """documents of more than CTA_MIN structurals, alone and in a stream between short ones: targets at the start, the
    middle and the end, keys first and last, misses that scan the whole container"""
    arr = long_array(3000)  # ~ 3000 * 10 structurals
    obj = json.dumps({f"k{i}": ([i] * (i % 4) if i % 2 else {"x": i}) for i in range(4000)}).encode()
    big = bytes(corpus.random_json(2 << 20, seed=77))
    for doc in (arr, obj, big):
        v = json.loads(doc)
        m = len(v)
        ptrs = ["", "/0", f"/{m // 2}", f"/{m - 1}", f"/{m}", "/-", "/k0", f"/k{m // 2}", f"/k{m - 1}", f"/k{m}", f"/{m - 1}/v/1", f"/{m - 2}/i",
                f"/k{m - 1}/x", f"/k{m - 2}/0", "/no"]
        r = O.Port().stage1(doc)
        assert r.n > CTA_MIN
        check(parser, doc, ptrs)
        check(parser, b"[1]\n" + doc + b'\n{"a":2}\n' + doc, ptrs + ["/a"], stream=True)


def test_bad_tables_limits_and_fenced_output(parser):
    doc = b'{"a":1}\n[2,3]\n{"a":{"b":4}}\n'
    d, res, d_type, d_payload, d_strbuf = device_tokens(parser, doc)
    n = parser.n_structural_indexes
    L = sj.lib()

    def call(table, ndocs, ptrs, out):
        enc = [q.encode() for q in ptrs]
        bufs = [C.create_string_buffer(e, len(e)) for e in enc]
        pp = (C.c_void_p * max(len(enc), 1))(*[C.addressof(b) for b in bufs])
        ll = (C.c_size_t * max(len(enc), 1))(*[len(e) for e in enc])
        return L.sjb200_at_pointer_dev(parser._ctx, d_type.data_ptr(), d_payload.data_ptr(), n, d_strbuf.data_ptr(), res.string_bytes,
                                       None if table is None else table.data_ptr(), ndocs, pp, ll, len(enc), out, None)

    # entries: ok, not ascending, ok, ok, >= n
    table = torch.tensor([0, 0, 0, 0, 7, 0, 8, 0, n, 0], dtype=torch.int32, device="cuda")
    ptrs = ["/a", "/0", ""]
    guard = 16
    fence = torch.full((2 * (guard + 5 * len(ptrs) + guard),), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    assert call(table, 5, ptrs, fence.data_ptr() + 8 * guard) == 0
    f = fence.cpu().numpy()
    assert (f[: 2 * guard] == 0x5A5A5A5A).all() and (f[2 * (guard + 15):] == 0x5A5A5A5A).all()
    res_ = f[2 * guard: 2 * (guard + 15)].reshape(3, 5, 2)
    assert res_[:, 1, 0].tolist() == [24] * 3 and res_[:, 4, 0].tolist() == [24] * 3
    assert res_[0, 0].tolist() == [0, 3] and res_[1, 2, 0] == 20 and res_[2, 3].tolist() == [0, 8]
    # limits: CAPACITY before any launch, nothing written
    out = torch.full((2 * 4,), 7, dtype=torch.int32, device="cuda")
    assert call(None, 0, ["/" + "/".join(["a"] * (capi.POINTER_MAX_TOKENS + 1))], out.data_ptr()) == sj.CAPACITY
    assert call(None, 0, ["/" + "a" * capi.POINTER_MAX_BYTES], out.data_ptr()) == sj.CAPACITY
    assert call(None, 0, ["/a"] * (capi.POINTER_MAX_POINTERS + 1), out.data_ptr()) == sj.CAPACITY
    assert (out.cpu() == 7).all()
    # n = 0: no document
    e, i = parser.at_pointer_device(["", "/a"], d_type[:0], d_payload[:0], d_strbuf, 0)
    assert e.cpu().tolist() == [[24], [24]]
