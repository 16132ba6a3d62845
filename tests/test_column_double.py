"""sjb200_column_double_dev on the H100 against the get_double oracle (sjo_double, pinned to the reference's
element::get_double and to float() by tests/test_double_oracle.py), bit for bit as uint64: the amazon rows at /5 (a mix
of 'l' and 'd'), the typed-column documents (1e400 is a 'd' row with NUMBER_ERROR), seeded float-heavy NDJSON rows with
the device document table, a column where one row in 16 takes the exact comparison, a row holding a 16 MiB number,
hand-made rows, fenced outputs, no rows and NULL outputs."""
import ctypes as C

import numpy as np
import pytest
import torch

import column_cases as CC
import double_cases as DC
import double_oracle as DO
import oracle_lib as O
import pointer_cases as PC
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
    res, d_type, d_payload, _d_strbuf = p.tokens_device(d)
    return d, res, d_type, d_payload, _d_strbuf


def device_table(p, d, n):
    table = torch.zeros(2 * (n + 8), dtype=torch.int32, device="cuda")
    nd = C.c_uint32(0)
    assert sj.lib().sjb200_document_table_dev(p._ctx, d.data_ptr(), p.device_index_buffer().data_ptr(), n, table.data_ptr(), n + 8, C.byref(nd), None) == 0
    return table, nd.value


def u64(t):
    return t.contiguous().view(torch.int64).cpu().numpy().ravel().view(np.uint64)


def check(p, doc, pointers, stream=False):
    """get_double of every pointer in every document against the oracle over the same rows; (err, type, bits, rows)"""
    d, res, d_type, d_payload, d_strbuf = device_tokens(p, doc)
    port = O.Port()
    r = port.stage1(doc)
    tw = port.tokens(doc, r.idx, r.n)
    if stream:
        table, nd = device_table(p, d, p.n_structural_indexes)
        perr, pidx = p.at_pointer_device(pointers, d_type, d_payload, d_strbuf, res.string_bytes, d_docs=table, ndocs=nd)
    else:
        perr, pidx = p.at_pointer_device(pointers, d_type, d_payload, d_strbuf, res.string_bytes)
    e, t, v = p.column_double_device(d, d_type, d_payload, perr, pidx)
    assert e.shape == t.shape == v.shape == perr.shape and v.dtype == torch.float64
    re_ = perr.cpu().numpy().ravel()
    ri = pidx.cpu().numpy().ravel().view(np.uint32)
    we, wt, wb = DO.Doubles().column(doc, r.idx[: r.n], tw[1], tw[2], re_, ri)
    ge, gt, gb = e.cpu().numpy().ravel(), t.cpu().numpy().ravel(), u64(v)
    bad = np.flatnonzero((ge != we) | (gt != wt) | (gb != wb))
    assert len(bad) == 0, [(int(i), int(ge[i]), int(we[i]), chr(gt[i]) if gt[i] else 0, hex(int(gb[i])), hex(int(wb[i]))) for i in bad[:6]]
    return ge, gt, gb, perr


def test_amazon_rows(parser):
    """the ratings at /5 mix 'l' and 'd'; /7 is an integer count, /0 a string"""
    e, t, _b, _perr = check(parser, PC.stream_of(PC.amazon_rows(100000)), ["/5", "/7", "/0", "/9"], stream=True)
    P = len(t) // 4
    kinds = set(t[:P].tolist())
    assert ord("l") in kinds and ord("d") in kinds
    assert (e[2 * P: 3 * P] == capi.INCORRECT_TYPE).all() and (e[3 * P:] == capi.INDEX_OUT_OF_BOUNDS).any()


def test_column_documents(parser):
    for _name, doc, pointers in CC.documents():
        check(parser, doc, pointers)
    e, t, b, _perr = check(parser, CC.INFINITE, ["/big", "/x"])
    assert (int(e[0]), int(t[0]), int(b[0])) == (DC.INF_ERROR, ord("d"), 0) and (int(e[1]), int(t[1])) == (0, ord("l"))
    e, t, b, _perr = check(parser, CC.EDGES, CC.EDGE_POINTERS)
    got = dict(zip(CC.EDGE_POINTERS, zip(e.tolist(), t.tolist(), b.tolist())))
    assert got["/nzero"] == (0, ord("l"), 0) and got["/half"] == (0, ord("d"), DC.bits(1.5)) and got["/umax"][2] == DC.bits(2.0 ** 64)
    assert got["/min"][2] == DC.bits(-2.0 ** 63) and got["/t"][0] == capi.INCORRECT_TYPE and got["/missing"][0] == capi.NO_SUCH_FIELD


def float_rows(texts, seed):
    rng = np.random.default_rng(seed)
    rows = []
    for i, x in enumerate(texts):
        y = texts[int(rng.integers(0, len(texts)))]
        rows.append(f'{{"a":{x},"b":{i},"c":[{y},{i % 7}],"s":"r{i}"}}'.encode())
    return rows


def test_float_rows(parser):
    """named cases and seeded numbers in NDJSON rows, with the device document table"""
    texts = DC.named_cases() + DC.random_numbers(200_000, 21)
    e, t, _b, _perr = check(parser, PC.stream_of(float_rows(texts, 5)), ["/a", "/b", "/c/0", "/c/1", "/s", "/c"], stream=True)
    assert (t == ord("d")).sum() > 200_000 and (e == DC.INF_ERROR).sum() > 0


def test_slow_path_column(parser):
    """one row in 16 is a halfway point written out exactly (or one unit off it): inconclusive for Eisel-Lemire"""
    rng = np.random.default_rng(3)
    xs = rng.integers(1, 2 ** 62, size=4096, dtype=np.int64).view(np.float64)
    texts = []
    for i, x in enumerate(xs[: 4096]):
        if not np.isfinite(x) or x == 0:
            x = 1.25
        texts.append(DC.halfway(float(x)) if i % 16 == 0 else repr(float(x)))
    texts[16] = DC.bump_last(texts[16], 1)
    texts[32] = DC.bump_last(texts[32], -1)
    rows = [f'{{"v":{x}}}'.encode() for x in texts]
    e, t, b, _perr = check(parser, PC.stream_of(rows), ["/v"], stream=True)
    want = np.array([DC.expect(x)[1] for x in texts], dtype=np.uint64)
    assert (e == 0).all() and np.array_equal(b, want)


def test_16mib_number(parser):
    """a row holding a 16 MiB number among short ones: summarized by a CTA; its 769th and later digits are a sticky bit"""
    h = DC.halfway(1.0)
    big = h + "0" * ((16 << 20) - len(h)) + "1"  # rounds up only because of its last digit
    rows = [b'{"v":1.5}', b'{"v":' + big.encode() + b'}', b'{"v":-0.0}', b'{"v":' + ("0." + "0" * 1000 + "25e1003").encode() + b'}']
    e, t, b, _perr = check(parser, PC.stream_of(rows), ["/v"], stream=True)
    assert e.tolist() == [0] * 4 and b.tolist() == [DC.bits(1.5), DC.bits(float(h)) + 1, DC.bits(-0.0), DC.bits(250.0)]


def raw(p, d, n, rows, nrows, err, rt, vals, d_type, d_payload, d_idx=None, length=None, out=None):
    res = capi.ColumnResult() if out is None else out
    rc = sj.lib().sjb200_column_double_dev(p._ctx, d.data_ptr(), d.numel() if length is None else length,
                                           (p.device_index_buffer() if d_idx is None else d_idx).data_ptr(), d_type.data_ptr(), d_payload.data_ptr(), n,
                                           rows, nrows, err, rt, vals, C.byref(res), None)
    return rc, res


def test_hand_made_rows_and_fenced_outputs(parser):
    doc = b'{"a":[1.25,-7,"x",{"b":2e-3}],"c":1e400,"d":18446744073709551615,"e":true,"f":3.5}'
    d, res, d_type, d_payload, _s = device_tokens(parser, doc)
    port = O.Port()
    r = port.stage1(doc)
    tw = port.tokens(doc, r.idx, r.n)
    types = bytes(tw[1])
    n = len(types)
    ds = [k for k, c in enumerate(types) if c == ord("d")]
    # a 'd' token whose payload is corrupted: past len, and an empty span
    payload = d_payload.clone()
    pl = tw[2].copy()
    for k, v in ((ds[0], len(doc) + 5), (ds[1], int(r.idx[ds[1]]))):
        payload[k] = v
        pl[k] = v
    rerr = [20, 0, 0, 0, 0] + [0] * n
    ridx = [0xFFFFFFFF, n + 5, types.index(b","), types.index(b":"), types.index(b"}")] + list(range(n))
    R = len(rerr)
    rows = torch.tensor(np.stack([np.array(rerr, dtype=np.int64), np.array(ridx, dtype=np.int64)], -1).astype(np.uint32).view(np.int32), device="cuda")
    we, wt, wb = DO.Doubles().column(doc, r.idx[: r.n], tw[1], pl, rerr, ridx)
    g = 64
    fe = torch.full((4 * R + 2 * g,), GUARD, dtype=torch.uint8, device="cuda")
    ft = torch.full((R + 2 * g,), GUARD, dtype=torch.uint8, device="cuda")
    fv = torch.full((8 * R + 2 * g,), GUARD, dtype=torch.uint8, device="cuda")
    rc, out = raw(parser, d, n, rows.data_ptr(), R, fe.data_ptr() + g, ft.data_ptr() + g, fv.data_ptr() + g, d_type, payload)
    assert rc == 0 and out.rows_in_error == int((we != 0).sum()) and out.string_bytes == 0
    for f, used in ((fe, 4 * R), (ft, R), (fv, 8 * R)):
        h = f.cpu().numpy()
        assert (h[:g] == GUARD).all() and (h[g + used:] == GUARD).all()
    e = fe[g: g + 4 * R].view(torch.int32).cpu().numpy()
    t = ft[g: g + R].cpu().numpy()
    v = fv[g: g + 8 * R].view(torch.int64).cpu().numpy().view(np.uint64)
    assert e.tolist() == we.tolist() and t.tolist() == wt.tolist() and v.tolist() == wb.tolist()
    assert e[:5].tolist() == [20, 24, 24, 24, 24] and t[:5].tolist() == [0] * 5
    assert (e[5 + ds[0]], t[5 + ds[0]]) == (24, 0) and (e[5 + ds[1]], t[5 + ds[1]]) == (24, 0)
    assert e[5 + ds[2]] == DC.INF_ERROR and v[5 + ds[2]] == 0 and v[5 + ds[3]] == DC.bits(3.5) and v[5 + types.index(b"u")] == DC.bits(2.0 ** 64)
    # nrows = 0 writes nothing; a NULL output or input that is needed is UNEXPECTED_ERROR
    fe.fill_(GUARD)
    rc, out = raw(parser, d, n, None, 0, None, None, None, d_type, payload)
    assert rc == 0 and out.rows_in_error == 0
    rp, ep, tp, vp = rows.data_ptr(), fe.data_ptr(), ft.data_ptr(), fv.data_ptr()
    for args in ((None, R, ep, tp, vp), (rp, R, None, tp, vp), (rp, R, ep, None, vp), (rp, R, ep, tp, None)):
        assert raw(parser, d, n, *args, d_type, payload)[0] == sj.UNEXPECTED_ERROR
    assert sj.lib().sjb200_column_double_dev(parser._ctx, d.data_ptr(), d.numel(), None, d_type.data_ptr(), payload.data_ptr(), n, rp, R, ep, tp, vp,
                                             C.byref(capi.ColumnResult()), None) == sj.UNEXPECTED_ERROR
    assert sj.lib().sjb200_column_double_dev(parser._ctx, d.data_ptr(), d.numel(), parser.device_index_buffer().data_ptr(), d_type.data_ptr(),
                                             payload.data_ptr(), n, rp, R, ep, tp, vp, None, None) == sj.UNEXPECTED_ERROR
    assert (fe.cpu().numpy() == GUARD).all()
