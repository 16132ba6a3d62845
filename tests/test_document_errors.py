"""sjb200_document_errors_dev on the H100 against the grammar oracle (sjo_document_errors, pinned to the reference's
stage 2 by tests/test_document_errors_oracle.py) and the golden file: the corpora, the fuzz set as one stream and one
document at a time, ~256 MiB of NDJSON rows with corrupted rows, the 64 MiB random document intact and corrupted, deep
nesting, bad tables, n = 0, CAPACITY, fenced output, and consistency with sjb200_at_pointer_dev."""
import ctypes as C

import numpy as np
import pytest
import torch

import grammar_oracle as G
import oracle_lib as O
import pointer_cases as PC
import pointer_oracle as PO
import simdjson_b200 as sj
from simdjson_b200 import capi, corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def parser():
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(300 << 20)
    assert rc == sj.SUCCESS
    yield p
    p.close()


@pytest.fixture(scope="module")
def gram():
    return G.Grammar()


def device_tokens(p, doc):
    d = torch.frombuffer(bytearray(doc), dtype=torch.uint8).cuda()
    assert p.stage1_device(d, sj.REGULAR) == sj.SUCCESS
    res, d_type, d_payload, _ = p.tokens_device(d)
    return d, d_type, d_payload


def device_table(p, d, n):
    table = torch.zeros(2 * (n + 8), dtype=torch.int32, device="cuda")
    nd = C.c_uint32(0)
    assert sj.lib().sjb200_document_table_dev(p._ctx, d.data_ptr(), p.device_index_buffer().data_ptr(), n, table.data_ptr(), n + 8, C.byref(nd), None) == 0
    return table, nd.value


def run(p, doc, stream=False, max_depth=1024):
    """device verdicts (res, err, idx as numpy), and the document starts (None: one document)"""
    d, d_type, d_payload = device_tokens(p, doc)
    if stream:
        table, nd = device_table(p, d, p.n_structural_indexes)
        starts = table[: 2 * nd].view(-1, 2)[:, 0].cpu().numpy().tolist()
        res, e, i = p.document_errors_device(d_type, d_payload, d_docs=table, ndocs=nd, max_depth=max_depth)
    else:
        starts = None
        res, e, i = p.document_errors_device(d_type, d_payload, max_depth=max_depth)
    return res, e.cpu().numpy(), i.cpu().numpy().view(np.uint32), starts, d_type, d_payload


def check(p, g, doc, stream=False, max_depth=1024):
    res, err, idx, starts, _, _ = run(p, doc, stream, max_depth)
    tk = g.tokens(doc)
    assert tk is not None
    if stream:
        assert starts == PO.document_starts(doc, tk[0].idx, tk[0].n)
    we, wi = g.errors(tk[1], tk[2], starts, max_depth)
    bad = np.argwhere((err != we) | (idx != wi)).ravel()
    assert len(bad) == 0, [(int(k), int(err[k]), int(idx[k]), int(we[k]), int(wi[k])) for k in bad[:8]]
    nerr = int((we != 0).sum())
    assert res.ndocs_in_error == nerr
    assert res.first_doc_in_error == (int(np.argmax(we != 0)) if nerr else G.NONE)
    return err, idx


def test_golden(parser, gram):
    gold = G.load_golden()
    for case in gold["cases"]:
        doc = bytes.fromhex(case["doc"])
        res, err, idx, starts, _, _ = run(parser, doc, case["stream"], case["max_depth"])
        assert err.tolist() == case["errors"] and idx.tolist() == case["indexes"], case


def test_corpora(parser, gram):
    for name in ("twitter.json", "citm_catalog.json"):
        err, _ = check(parser, gram, O.jsonexample(name))
        assert err[0] == 0
    check(parser, gram, O.jsonexample("amazon_cellphones.ndjson"), stream=True)
    check(parser, gram, PC.stream_of(PC.twitter_rows()), stream=True)


def test_fuzz_set(parser, gram):
    docs = G.fuzz_docs(3000)
    check(parser, gram, b"\n".join(docs), stream=True)
    check(parser, gram, b"".join(docs), stream=True)
    for d in docs[:400]:
        check(parser, gram, d)


def test_ndjson_256m_with_corrupt_rows(parser, gram):
    rows = PC.twitter_rows()
    base = PC.stream_of(rows)
    reps = (256 << 20) // len(base)
    lines = (base * reps).split(b"\n")[:-1]
    bad_at = sorted({7, 1234, len(lines) // 2, len(lines) - 3, len(lines) - 1})
    for k in bad_at:
        lines[k] = lines[k].replace(b', "', b': "', 1) if k % 2 else lines[k][:-1] + b",}"
    doc = b"\n".join(lines) + b"\n"
    res, err, idx, starts, _, _ = run(parser, doc, stream=True)
    assert len(starts) == len(lines)
    assert res.ndocs_in_error == len(bad_at) and res.first_doc_in_error == bad_at[0]
    assert np.flatnonzero(err).tolist() == bad_at
    assert set(err[bad_at].tolist()) == {G.TAPE_ERROR}


def test_64m_document(parser, gram):
    big = bytearray(corpus.random_json(64 << 20, seed=5))
    check(parser, gram, bytes(big))
    r = O.Port().stage1(bytes(big))
    for frac in (0.001, 0.5, 0.999):
        k = int(r.n * frac)
        while big[r.idx[k]] != ord(","):
            k += 1
        doc = bytearray(big)
        doc[r.idx[k]] = ord(" ")
        err, _ = check(parser, gram, bytes(doc))
        assert err[0] != 0


def test_deep_nesting(parser, gram):
    one = G.nested(1000, b'{"a":[1,2,{}]}')
    doc = b"[" + b",".join([one] * 200) + b"]"
    err, _ = check(parser, gram, doc, max_depth=1024)
    assert err[0] == 0
    err, _ = check(parser, gram, doc, max_depth=1000)
    assert err[0] == G.DEPTH_ERROR
    check(parser, gram, b"\n".join([one] * 50 + [one[:-1]] + [one] * 50), stream=True)


def test_bad_tables_empty_capacity_and_fenced_output(parser, gram):
    doc = b'{"a":1}\n[2,3]\n{"a":{"b":4}}\n'
    d, d_type, d_payload = device_tokens(parser, doc)
    n = parser.n_structural_indexes
    L = sj.lib()
    guard = 16
    before = (d_type.clone(), d_payload.clone())

    def call(table, ndocs, out, max_depth=1024, t=d_type):
        res = capi.DocumentErrorsResult()
        rc = L.sjb200_document_errors_dev(parser._ctx, t.data_ptr(), d_payload.data_ptr(), t.numel(), None if table is None else table.data_ptr(), ndocs,
                                          max_depth, out, C.byref(res), None)
        return rc, res

    fence = torch.full((2 * (guard + 3 + guard),), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    good = torch.tensor([0, 0, 5, 0, 10, 0], dtype=torch.int32, device="cuda")
    rc, res = call(good, 3, fence.data_ptr() + 8 * guard)
    f = fence.cpu().numpy()
    assert rc == 0 and res.ndocs_in_error == 0 and res.first_doc_in_error == G.NONE
    assert (f[: 2 * guard] == 0x5A5A5A5A).all() and (f[2 * (guard + 3):] == 0x5A5A5A5A).all()
    assert f[2 * guard: 2 * (guard + 3)].tolist() == [0, 5, 0, 10, 0, n]
    assert torch.equal(before[0], d_type) and torch.equal(before[1], d_payload)
    # not ascending, and an entry at or above n: UNEXPECTED_ERROR everywhere
    for bad in ([0, 0, 5, 0, 5, 0], [0, 0, 5, 0, n, 0], [3, 0, 1, 0, 10, 0]):
        out = torch.full((6,), 7, dtype=torch.int32, device="cuda")
        rc, res = call(torch.tensor(bad, dtype=torch.int32, device="cuda"), 3, out.data_ptr())
        assert rc == sj.UNEXPECTED_ERROR and out.cpu().view(-1, 2).tolist() == [[24, -1]] * 3 and res.ndocs_in_error == 3
    # CAPACITY before any launch, nothing written
    out = torch.full((6,), 7, dtype=torch.int32, device="cuda")
    for md in (0, capi.DOCUMENT_MAX_DEPTH + 1):
        assert call(good, 3, out.data_ptr(), md)[0] == sj.CAPACITY
    assert (out.cpu() == 7).all()
    # n = 0: EMPTY
    rc, res = call(None, 0, out.data_ptr(), t=d_type[:0])
    assert rc == 0 and out.cpu()[:2].tolist() == [13, 0] and res.ndocs_in_error == 1 and res.first_doc_in_error == 0


def test_at_pointer_consistency(parser, gram):
    """documents whose verdict is SUCCESS: at_pointer as the reference's; the others: the verdict is the parse error"""
    docs = G.fuzz_docs(400, seed=3)
    doc = b"\n".join(docs)
    d = torch.frombuffer(bytearray(doc), dtype=torch.uint8).cuda()
    assert parser.stage1_device(d, sj.REGULAR) == sj.SUCCESS
    res, d_type, d_payload, d_strbuf = parser.tokens_device(d)
    n = parser.n_structural_indexes
    table, nd = device_table(parser, d, n)
    _, err, idx = parser.document_errors_device(d_type, d_payload, d_docs=table, ndocs=nd)
    ptrs = ["", "/0", "/user/id", "/1"]
    perr, pidx = parser.at_pointer_device(ptrs, d_type, d_payload, d_strbuf, res.string_bytes, d_docs=table, ndocs=nd)
    err, perr, pidx = err.cpu().numpy(), perr.cpu().numpy(), pidx.cpu().numpy().view(np.uint32)
    starts = table[: 2 * nd].view(-1, 2)[:, 0].cpu().numpy().tolist()
    r = O.Port().stage1(doc)
    pto = PO.Pointers()
    tw = O.Port().tokens(doc, r.idx, r.n)
    ok = 0
    for k, s in enumerate(starts):
        end = starts[k + 1] if k + 1 < len(starts) else n
        if err[k] == 0:
            ok += 1
            for p, q in enumerate(ptrs):
                assert (int(perr[p, k]), int(pidx[p, k])) == pto.at_pointer(tw[1], tw[2], tw[3], q, s, end)
    assert ok > 50
