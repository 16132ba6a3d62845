"""sjb200_column_dev on the H100 against the typed-column oracle (sjo_column, pinned to the reference's DOM getters by
tests/test_column_oracle.py): every kind -- get_int64, get_uint64, get_bool, get_string, get_array().size(),
get_object().size() -- on the results of sjb200_at_pointer_dev for twitter NDJSON rows with the device document table,
the pointer corpora, integer edges, floats, atoms, strings of every length around the vector width and of 1 MiB,
containers walked by a warp and by a CTA, an array past the tape count's saturation, hand-made rows, fenced outputs, the
CAPACITY round trip and no rows."""
import ctypes as C

import numpy as np
import pytest
import torch

import column_cases as CC
import column_oracle as CO
import oracle_lib as O
import pointer_cases as PC
import pointer_oracle as PO
import simdjson_b200 as sj
from simdjson_b200 import capi

pytestmark = pytest.mark.gpu

GUARD = 0x5A


@pytest.fixture(scope="module")
def parser():
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(64 << 20)
    assert rc == sj.SUCCESS
    yield p
    p.close()


def device_tokens(p, doc):
    d = torch.frombuffer(bytearray(doc), dtype=torch.uint8).cuda()
    assert p.stage1_device(d, sj.REGULAR) == sj.SUCCESS
    res, d_type, d_payload, d_strbuf = p.tokens_device(d)
    return d, res, d_type, d_payload, d_strbuf


def device_table(p, d, n):
    table = torch.zeros(2 * (n + 8), dtype=torch.int32, device="cuda")
    nd = C.c_uint32(0)
    assert sj.lib().sjb200_document_table_dev(p._ctx, d.data_ptr(), p.device_index_buffer().data_ptr(), n, table.data_ptr(), n + 8, C.byref(nd), None) == 0
    return table, nd.value


def host_tokens(doc):
    port = O.Port()
    r = port.stage1(doc)
    return r, port.tokens(doc, r.idx, r.n)


def strings_of(offsets, data):
    o = offsets.cpu().numpy()
    b = bytes(data.cpu().numpy())
    return [b[o[i]: o[i + 1]] for i in range(len(o) - 1)]


def check_rows(p, tok, tw, perr, pidx, kinds=CO.KINDS):
    """every kind over device rows (perr, pidx) against the oracle over the same rows"""
    _d, res, d_type, d_payload, d_strbuf = tok
    cols = CO.Columns()
    re_ = perr.cpu().numpy().ravel()
    ri = pidx.cpu().numpy().ravel().view(np.uint32)
    for kind in kinds:
        we, wt, wv, ws = cols.column(kind, tw[1], tw[2], tw[3], len(tw[3]), re_, ri)
        out = p.column_device(kind, d_type, d_payload, d_strbuf, res.string_bytes, perr, pidx)
        assert out[0].shape == perr.shape
        e, t = out[0].cpu().numpy().ravel(), out[1].cpu().numpy().ravel()
        bad = np.flatnonzero((e != we) | (t != wt))
        assert len(bad) == 0, (kind, [(int(i), int(e[i]), int(we[i]), int(t[i]), int(wt[i])) for i in bad[:6]])
        if kind == CO.STRING:
            got = strings_of(out[2], out[3])
            assert int(out[2][-1]) == sum(len(s) for s in ws)
            bad = [i for i in range(len(ws)) if got[i] != ws[i]]
            assert not bad, (kind, bad[:6])
        else:
            v = out[2].cpu().numpy().ravel()
            v = v.astype(np.uint64) if kind == CO.BOOL else v.view(np.uint64)
            bad = np.flatnonzero(v != wv)
            assert len(bad) == 0, (kind, [(int(i), int(v[i]), int(wv[i])) for i in bad[:6]])


def check(p, doc, pointers, stream=False, kinds=CO.KINDS):
    tok = device_tokens(p, doc)
    _d, res, d_type, d_payload, d_strbuf = tok
    _r, tw = host_tokens(doc)
    if stream:
        table, nd = device_table(p, tok[0], p.n_structural_indexes)
        perr, pidx = p.at_pointer_device(pointers, d_type, d_payload, d_strbuf, res.string_bytes, d_docs=table, ndocs=nd)
    else:
        perr, pidx = p.at_pointer_device(pointers, d_type, d_payload, d_strbuf, res.string_bytes)
    check_rows(p, tok, tw, perr, pidx, kinds)
    return tok, tw, perr, pidx


def test_twitter_rows(parser):
    tok, _tw, perr, pidx = check(parser, PC.stream_of(PC.twitter_rows()), CC.TWITTER_POINTERS, stream=True)
    e = perr.cpu().numpy()
    assert (e[0] == 0).all() and (e[-1] != 0).sum() > 0  # /retweeted_status/id is missing from most rows
    # one pointer's row of the pair, and rows that are not views of one pair tensor (one packing copy)
    _d, res, d_type, d_payload, d_strbuf = tok
    ids = parser.column_device(capi.COLUMN_INT64, d_type, d_payload, d_strbuf, res.string_bytes, perr[1], pidx[1])
    again = parser.column_device(capi.COLUMN_INT64, d_type, d_payload, d_strbuf, res.string_bytes, perr[1].clone(), pidx[1].clone())
    allp = parser.column_device(capi.COLUMN_INT64, d_type, d_payload, d_strbuf, res.string_bytes, perr, pidx)
    for a, b, c in zip(ids, again, allp):
        assert torch.equal(a, b) and torch.equal(a, c[1])


def test_pointer_corpora(parser):
    for name, doc, pointers in PC.corpus_cases(full=False):
        check(parser, doc, pointers[:300] + pointers[-40:])


def test_column_documents(parser):
    """integer edges, floats, atoms under every kind; strings; containers (empty, duplicate keys, longer than the warp
    walk's limit and than one CTA step)"""
    for name, doc, pointers in CC.documents():
        check(parser, doc, pointers)
    docs = [d for n, d, _p in CC.documents()]
    check(parser, b"\n".join(docs) + b"\n", sorted({q for _n, _d, ps in CC.documents() for q in ps}), stream=True)
    # the edges' values themselves
    tok, _tw, perr, pidx = check(parser, CC.EDGES, CC.EDGE_POINTERS)
    _d, res, d_type, d_payload, d_strbuf = tok
    e, t, v = parser.column_device(capi.COLUMN_INT64, d_type, d_payload, d_strbuf, res.string_bytes, perr, pidx)
    got = dict(zip(CC.EDGE_POINTERS, zip(e[:, 0].tolist(), v[:, 0].tolist(), t[:, 0].tolist())))
    assert got["/min"] == (0, -2 ** 63, ord("l")) and got["/max"] == (0, 2 ** 63 - 1, ord("l"))
    assert got["/over"][:2] == (capi.NUMBER_OUT_OF_RANGE, 0) and got["/nzero"] == (0, 0, ord("l"))
    assert got["/half"] == (capi.INCORRECT_TYPE, 0, ord("d")) and got["/missing"][:2] == (capi.NO_SUCH_FIELD, 0)
    e, t, v = parser.column_device(capi.COLUMN_UINT64, d_type, d_payload, d_strbuf, res.string_bytes, perr, pidx)
    got = dict(zip(CC.EDGE_POINTERS, zip(e[:, 0].tolist(), v[:, 0].tolist())))
    assert got["/umax"] == (0, -1) and got["/m1"] == (capi.NUMBER_OUT_OF_RANGE, 0) and got["/over"] == (0, -2 ** 63)


def test_infinite_float_is_a_d_row(parser):
    """1e400: the reference's parse fails (the value is infinite), but the tokens only check float grammar -- the
    inherited deviation of sjb200_tokens_dev -- so here the row is a 'd' value, INCORRECT_TYPE under every kind"""
    tok, _tw, perr, pidx = check(parser, CC.INFINITE, ["/big", "/x"])
    _d, res, d_type, d_payload, d_strbuf = tok
    for kind in CO.KINDS:
        out = parser.column_device(kind, d_type, d_payload, d_strbuf, res.string_bytes, perr, pidx)
        assert (int(out[0][0, 0]), int(out[1][0, 0])) == (capi.INCORRECT_TYPE, ord("d"))


def test_long_strings(parser):
    """a 1 MiB string between short ones, strings copied by a lane, a warp and several CTAs, in staged and direct tiles"""
    import json
    rng = np.random.default_rng(5)
    big = "".join(chr(c) for c in rng.integers(0x20, 0x7F, 1 << 20)).replace("\\", "/").replace('"', "'")
    vals = ["s", big, "t", "u" * 5000, "v" * 70000, "w" * 31, "x" * 33, "é" * 3000] + [f"r{i}" * (i % 40) for i in range(600)]
    rows = [json.dumps({"k": v, "i": i}, ensure_ascii=False).encode() for i, v in enumerate(vals)]
    check(parser, PC.stream_of(rows), ["/k", "/i", ""], stream=True, kinds=(CO.STRING, CO.INT64, CO.OBJECT_SIZE))


def test_many_long_strings(parser):
    """a column where most strings are over the warp's 4 KiB: each is listed chunk by chunk (one to three 16 KiB chunks)
    and copied by the CTAs of the long-string kernel, next to short ones in the same tiles"""
    import json
    rng = np.random.default_rng(9)
    pool = "".join(chr(c) for c in rng.integers(0x20, 0x7F, 64 << 10)).replace("\\", "/").replace('"', "'")
    lens = rng.integers(4000, 40000, 1200)
    vals = [pool[int(o): int(o) + int(n)] if i % 7 else f"s{i}" for i, (o, n) in enumerate(zip(rng.integers(0, 20000, len(lens)), lens))]
    rows = [json.dumps({"b": v}).encode() for v in vals]
    check(parser, PC.stream_of(rows), ["/b"], stream=True, kinds=(CO.STRING,))


def test_size_saturates(parser):
    doc = CC.big_array(16777216)
    tok = device_tokens(parser, doc)
    _d, res, d_type, d_payload, d_strbuf = tok
    perr, pidx = parser.at_pointer_device(["", "/16777215"], d_type, d_payload, d_strbuf, res.string_bytes)
    e, t, v = parser.column_device(capi.COLUMN_ARRAY_SIZE, d_type, d_payload, d_strbuf, res.string_bytes, perr, pidx)
    assert e[:, 0].tolist() == [0, capi.INCORRECT_TYPE] and v[0, 0].item() == 0xFFFFFF and t[0, 0].item() == ord("[")


def raw(p, kind, tok, rows, nrows, err, rt, vals, offs, data, cap, string_bytes=None):
    _d, res, d_type, d_payload, d_strbuf = tok
    out = capi.ColumnResult()
    sb = res.string_bytes if string_bytes is None else string_bytes
    rc = sj.lib().sjb200_column_dev(p._ctx, kind, d_type.data_ptr(), d_payload.data_ptr(), d_type.numel(), d_strbuf.data_ptr(), sb,
                                    rows, nrows, err, rt, vals, offs, data, cap, C.byref(out), None)
    return rc, out


def test_hand_made_rows_and_fenced_outputs(parser):
    doc = b'{"a":[1,"xyz",{"b":true}],"c":"","d":"0123456789abcdefghij"}'
    tok = device_tokens(parser, doc)
    _r, tw = host_tokens(doc)
    types = bytes(tw[1])
    n = len(types)
    strs = [k for k, t in enumerate(types) if t == ord('"') and (k + 1 >= n or types[k + 1] != ord(":"))]
    # rows: in error, past n, at ',' and '}', then every value
    rerr = [20, 0, 0, 0] + [0] * n
    ridx = [0xFFFFFFFF, n + 5, types.index(b","), types.index(b"}"), ] + list(range(n))
    keep = [i for i in range(len(rerr)) if i < 4 or types[ridx[i]] not in b",:}]"]
    rerr, ridx = [rerr[i] for i in keep] + [0, 0], [ridx[i] for i in keep] + strs[:2]
    R = len(rerr)
    rows = torch.tensor(np.stack([np.array(rerr, dtype=np.int64), np.array(ridx, dtype=np.int64)], -1).astype(np.uint32).view(np.int32), device="cuda")
    cols = CO.Columns()
    g = 64  # guard bytes on each side of every output
    for kind in CO.KINDS:
        we, wt, wv, ws = cols.column(kind, tw[1], tw[2], tw[3], len(tw[3]), rerr, ridx)
        fe = torch.full((4 * R + 2 * g,), GUARD, dtype=torch.uint8, device="cuda")
        ft = torch.full((R + 2 * g,), GUARD, dtype=torch.uint8, device="cuda")
        vb = 1 if kind == CO.BOOL else 8
        fv = torch.full((vb * R + 2 * g,), GUARD, dtype=torch.uint8, device="cuda")
        fo = torch.full((8 * (R + 1) + 2 * g,), GUARD, dtype=torch.uint8, device="cuda")
        need = sum(len(s) for s in ws)
        fb = torch.full((need + 2 * g + 37,), GUARD, dtype=torch.uint8, device="cuda")
        st = kind == CO.STRING
        rc, out = raw(parser, kind, tok, rows.data_ptr(), R, fe.data_ptr() + g, ft.data_ptr() + g, None if st else fv.data_ptr() + g,
                      fo.data_ptr() + g if st else None, fb.data_ptr() + g + 3 if st else None, need + 37 if st else 0)
        assert rc == 0 and out.rows_in_error == int((we != 0).sum())
        for f, used in ((fe, 4 * R), (ft, R), (fv, 0 if st else vb * R), (fo, 8 * (R + 1) if st else 0), (fb, need + 3 if st else 0)):
            h = f.cpu().numpy()
            inner = slice(g, g + used) if f is not fb else slice(g + 3, g + used)
            outside = np.ones(len(h), dtype=bool)
            outside[inner] = False
            assert (h[outside] == GUARD).all(), (kind, np.flatnonzero(h[outside] != GUARD)[:8])
        e = fe[g: g + 4 * R].view(torch.int32).cpu().numpy()
        t = ft[g: g + R].cpu().numpy()
        assert e.tolist() == we.tolist() and t.tolist() == wt.tolist(), kind
        assert e[:4].tolist() == [20, 24, 24, 24] and t[:4].tolist() == [0] * 4
        if st:
            offs = fo[g: g + 8 * (R + 1)].view(torch.int64)
            assert out.string_bytes == need and strings_of(offs, fb[g + 3: g + 3 + need]) == ws
        else:
            v = fv[g: g + vb * R]
            v = v.cpu().numpy().astype(np.uint64) if vb == 1 else v.view(torch.int64).cpu().numpy().view(np.uint64)
            assert v.tolist() == wv.tolist(), kind
    # a string_bytes that cuts the string buffer short: a STRING row whose record does not lie inside it is
    # UNEXPECTED_ERROR with row type 0, the others keep their strings; under INT64 the record is not read
    for cut in (0, 3, 7, 12, len(tw[3]) - 1):
        for kind in (CO.STRING, CO.INT64):
            we, wt, wv, ws = cols.column(kind, tw[1], tw[2], tw[3][:cut], cut, rerr, ridx)
            e = torch.empty(R, dtype=torch.int32, device="cuda")
            t = torch.empty(R, dtype=torch.uint8, device="cuda")
            o = torch.empty(R + 1, dtype=torch.int64, device="cuda")
            v = torch.empty(R, dtype=torch.int64, device="cuda")
            b = torch.empty(len(tw[3]) + 16, dtype=torch.uint8, device="cuda")
            st = kind == CO.STRING
            rc, out = raw(parser, kind, tok, rows.data_ptr(), R, e.data_ptr(), t.data_ptr(), None if st else v.data_ptr(), o.data_ptr() if st else None,
                          b.data_ptr() if st else None, b.numel() if st else 0, string_bytes=cut)
            assert rc == 0 and out.rows_in_error == int((we != 0).sum())
            assert e.cpu().tolist() == we.tolist() and t.cpu().tolist() == wt.tolist(), (cut, kind)
            if st:
                assert strings_of(o, b[: out.string_bytes]) == ws, cut
                assert (we == 24).sum() >= 4  # the three hand-made rows and at least the last string


def test_capacity_round_trip_and_no_rows(parser):
    doc = PC.stream_of(PC.twitter_rows())
    tok = device_tokens(parser, doc)
    _d, res, d_type, d_payload, d_strbuf = tok
    table, nd = device_table(parser, tok[0], parser.n_structural_indexes)
    perr, pidx = parser.at_pointer_device(["/text"], d_type, d_payload, d_strbuf, res.string_bytes, d_docs=table, ndocs=nd)
    rows = torch.stack((perr[0], pidx[0]), -1).contiguous()
    R = rows.shape[0]
    e = torch.empty(R, dtype=torch.int32, device="cuda")
    t = torch.empty(R, dtype=torch.uint8, device="cuda")
    o = torch.empty(R + 1, dtype=torch.int64, device="cuda")
    rc, out = raw(parser, capi.COLUMN_STRING, tok, rows.data_ptr(), R, e.data_ptr(), t.data_ptr(), None, o.data_ptr(), None, 0)
    need = out.string_bytes
    assert rc == sj.CAPACITY and need > 0
    want_offs = o.clone()
    b = torch.full((need + 16,), GUARD, dtype=torch.uint8, device="cuda")
    rc, out = raw(parser, capi.COLUMN_STRING, tok, rows.data_ptr(), R, e.data_ptr(), t.data_ptr(), None, o.data_ptr(), b.data_ptr(), need - 1)
    assert rc == sj.CAPACITY and out.string_bytes == need and (b.cpu() == GUARD).all() and torch.equal(o, want_offs)
    rc, out = raw(parser, capi.COLUMN_STRING, tok, rows.data_ptr(), R, e.data_ptr(), t.data_ptr(), None, o.data_ptr(), b.data_ptr(), need)
    assert rc == 0 and out.string_bytes == need and (b[need:].cpu() == GUARD).all() and torch.equal(o, want_offs)
    _e, _t, offs, data = parser.column_device(capi.COLUMN_STRING, d_type, d_payload, d_strbuf, res.string_bytes, perr, pidx)
    assert torch.equal(data, b[:need]) and torch.equal(offs, o)
    # nrows = 0: d_offsets[0] = 0 and nothing else
    o2 = torch.full((2,), 77, dtype=torch.int64, device="cuda")
    rc, out = raw(parser, capi.COLUMN_STRING, tok, None, 0, None, None, None, o2.data_ptr(), None, 0)
    assert rc == 0 and o2.tolist() == [0, 77] and (out.rows_in_error, out.string_bytes) == (0, 0)
    v2 = torch.full((2,), 77, dtype=torch.int64, device="cuda")
    rc, out = raw(parser, capi.COLUMN_INT64, tok, None, 0, None, None, v2.data_ptr(), None, None, 0)
    assert rc == 0 and v2.tolist() == [77, 77]
    # an unknown kind, a missing output
    assert raw(parser, 7, tok, rows.data_ptr(), R, e.data_ptr(), t.data_ptr(), o.data_ptr(), None, None, 0)[0] == sj.UNEXPECTED_ERROR
    assert raw(parser, capi.COLUMN_BOOL, tok, rows.data_ptr(), R, e.data_ptr(), t.data_ptr(), None, None, None, 0)[0] == sj.UNEXPECTED_ERROR
    assert raw(parser, capi.COLUMN_STRING, tok, rows.data_ptr(), R, e.data_ptr(), t.data_ptr(), None, None, None, 0)[0] == sj.UNEXPECTED_ERROR
