"""Pins the CPU restatement (oracle/sj_oracle.c) before anything trusts it.

 * against the committed golden vectors produced by the unmodified reference
   (tests/golden/*.json, generator oracle/gen_golden.py) -- runs everywhere;
 * against the live reference (oracle/_ref/libsj_ref.so: icelake AND haswell)
   on seeded adversarial inputs, all seven stage1 modes -- runs wherever the
   prebuilt reference .so is present (it ships to the GPU box too).
"""
import hashlib
import json
import os
import random

import numpy as np
import pytest

import oracle_lib as O
from simdjson_b200 import corpus

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def port():
    return O.Port()


def _load(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def test_port_matches_golden_stage1(port):
    cases = _load("stage1.json")["cases"]
    assert len(cases) > 500
    for c in cases:
        r = port.stage1(bytes.fromhex(c["hex"]), c["mode"])
        assert r.err == c["err"], c
        if c["n"] is None:
            assert not r.wrote, c
        else:
            assert r.n == c["n"], c
            assert [int(x) for x in r.words()] == c["words"], c


def test_port_matches_golden_minify(port):
    cases = _load("minify.json")["cases"]
    assert len(cases) > 400
    for c in cases:
        err, out = port.minify(bytes.fromhex(c["hex"]))
        assert (err, out.hex()) == (c["err"], c["out"]), c


def test_port_matches_golden_utf8(port):
    cases = _load("utf8.json")["cases"]
    assert len(cases) > 300
    for c in cases:
        assert port.validate_utf8(bytes.fromhex(c["hex"])) == c["valid"], c


def test_port_matches_golden_corpora(port):
    for f in _load("corpora.json")["files"]:
        data = np.frombuffer(O.jsonexample(f["file"]), dtype=np.uint8)
        assert len(data) == f["len"]
        r = port.stage1(data, f["mode"])
        assert (r.err, r.n) == (f["err"], f["n"])
        assert hashlib.sha256(r.words().tobytes()).hexdigest() == f["idx_sha256"]
        err, out = port.minify(data)
        assert (err, len(out), hashlib.sha256(out).hexdigest()) == (f["minify_err"], f["minify_len"], f["minify_sha256"])
        assert port.validate_utf8(data) == f["utf8"]


def test_amazon_is_793_documents(port):
    """tests/dom/basictests.cpp L36, L692-708: parse_many over amazon_cellphones.ndjson yields 793 docs;
    at stage-1 level: 793 top-level '[' ... ']' rows in streaming_final mode."""
    data = np.frombuffer(O.jsonexample("amazon_cellphones.ndjson"), dtype=np.uint8)
    r = port.stage1(data, O.STREAMING_FINAL)
    assert r.err == 0 and r.n == 15067
    # count row starts: a '[' structural that is the first structural on its line
    starts = 0
    idx = r.idx[: r.n]
    for k, pos in enumerate(idx):
        if data[pos] == ord("[") and (k == 0 or data[idx[k - 1]] == ord("]")):
            starts += 1
    assert starts == 793


needs_ref = pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref/libsj_ref.so not built")


@needs_ref
@pytest.mark.parametrize("impl", ["icelake", "haswell"])
def test_port_matches_live_reference_fuzz(port, impl):
    if impl not in O.ref_impls():
        pytest.skip(f"{impl} not supported by this host")
    ref = O.Ref(impl)
    rng = random.Random(corpus.SEED + (1 if impl == "haswell" else 0))
    n_cases = 4000
    for i in range(n_cases):
        kind = i % 4
        if kind == 0:
            b, mode = corpus.adversarial(rng), rng.choice(O.ALL_MODES)
        elif kind == 1:
            b, mode = corpus.multi_document(rng), rng.choice([1, 2])
        elif kind == 2:
            b, mode = b"\x1e" + corpus.multi_document(rng, sep=b"\x1e"), rng.choice([3, 4])
        else:
            b, mode = corpus.multi_document(rng, sep=b","), rng.choice([5, 6])
        a, r = port.stage1(b, mode), ref.stage1(b, mode)
        assert O.same_stage1(a, r), (b, mode, a.err, r.err, a.n, r.n)
        if kind == 0:
            assert port.minify(b) == ref.minify(b), b
            assert port.validate_utf8(b) == ref.validate_utf8(b), b


@needs_ref
def test_port_matches_live_reference_capacity_and_sizes(port):
    ref = O.Ref("")
    doc = b'{"a":[1,2,3],"b":"xyz"}'
    # len > capacity -> CAPACITY before anything is written (json_structural_indexer.h L195)
    a, r = port.stage1(doc, 0, capacity=8), ref.stage1(doc, 0, capacity=8)
    assert a.err == r.err == O.CAPACITY and not a.wrote and not r.wrote
    # block-boundary lengths
    rng = random.Random(5)
    for n in list(range(0, 200)) + [255, 256, 257, 4095, 4096, 4097]:
        b = bytes(corpus.random_json(max(n, 64)))[:n]
        for mode in (0, 1, 2):
            assert O.same_stage1(port.stage1(b, mode), ref.stage1(b, mode)), (n, mode)
        assert port.minify(b) == ref.minify(b)
        u = bytes(corpus.random_utf8(max(n, 1), seed=n))[:n]
        assert port.validate_utf8(u) == ref.validate_utf8(u), n
        _ = rng


@needs_ref
def test_port_matches_live_reference_large(port):
    ref = O.Ref("")
    d = corpus.random_json(4 << 20)
    assert O.same_stage1(port.stage1(d), ref.stage1(d))
    assert port.minify(d) == ref.minify(d)
    nd = corpus.ndjson_rows(2 << 20)
    for mode in (1, 2):
        assert O.same_stage1(port.stage1(nd, mode), ref.stage1(nd, mode))
    # cut an NDJSON buffer mid-row: streaming_partial must point at the last complete row
    cut = nd[: (1 << 20) + 123]
    a, r = port.stage1(cut, 1), ref.stage1(cut, 1)
    assert O.same_stage1(a, r) and a.err == 0 and a.idx[a.n] < len(cut)
    u = corpus.random_utf8(1 << 20)
    assert port.validate_utf8(u) and ref.validate_utf8(u)
    for pos in (0, len(u) // 2, len(u) - 2):
        v = u.copy()
        v[pos] = 0xFF
        assert not port.validate_utf8(v) and not ref.validate_utf8(v)


# ---------------------------------------------------------------- stage-2-lite (SURVEY.md 8(f) row 4)
import token_fuzz as TF  # noqa: E402


def _tape_view(types, pay):
    """the port's per-structural arrays in the reference's tape order: ':' and ',' have no tape entry"""
    keep = [i for i, t in enumerate(types) if chr(t) not in ":,"]
    return bytes(types[keep]), pay[keep]


def _check_doc_against(port, doc, want_err, want_types, want_pay_by_index, want_sb):
    r = port.stage1(doc)
    assert r.err == 0
    err, types, pay, sb, sl, ns, fe = port.tokens(doc, r.idx, r.n)
    assert err == 0 and fe == 0xFFFFFFFF, (doc[:80], err)
    t, p = _tape_view(types, pay)
    assert want_err == 0 and t == want_types, doc[:80]
    for i, v in want_pay_by_index.items():
        assert int(p[int(i)]) == int(v), (doc[:80], i)
    assert bytes(sb) == want_sb and sl == len(want_sb)


def test_port_tokens_match_golden(port):
    g = _load("tokens.json")
    for c in g["strings"]:
        body = bytes.fromhex(c["body"])
        r, out = port.parse_string(b'"' + body + b'"')
        assert r == c["len"] and out == bytes.fromhex(c["out"]), body
    for c in g["scalars"]:
        doc = bytes.fromhex(c["doc"])
        r = port.stage1(doc)
        if r.err != 0:  # stage 1 already fails (a quote inside the token): the reference reports the same error
            assert c["err"] == r.err, doc
            continue
        err, types, pay, *_ = port.tokens(doc, r.idx, r.n)
        k = c["index"]
        if c["err"] == 0:
            assert err == 0 and chr(types[k]) == c["type"], doc
            if c["value"] is not None:
                assert int(pay[k]) == int(c["value"]), doc
        else:
            # the reference stops at its first error; the token must be that error (it is the only scalar that can fail here)
            assert types[k] == 0 and int(pay[k]) == c["err"] and err == c["err"], (doc, err, int(pay[k]), c["err"])
    for c in g["documents"]:
        _check_doc_against(port, bytes.fromhex(c["doc"]), c["err"], c["types"].encode("latin1"), c["payloads"], bytes.fromhex(c["string_buf"]))
    for f in g["files"]:
        doc = O.jsonexample(f["file"])
        r = port.stage1(doc)
        err, types, pay, sb, sl, ns, fe = port.tokens(doc, r.idx, r.n)
        t, p = _tape_view(types, pay)
        assert err == 0 and len(t) == f["entries"] and hashlib.sha256(t).hexdigest() == f["types_sha256"]
        isd = np.frombuffer(t, dtype=np.uint8) == ord("d")
        assert hashlib.sha256(np.where(isd, 0, p).astype(np.uint64).tobytes()).hexdigest() == f["payloads_no_doubles_sha256"]
        assert sl == f["string_buf_bytes"] and hashlib.sha256(bytes(sb)).hexdigest() == f["string_buf_sha256"]


@pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref/libsj_ref.so not built")
def test_port_tokens_match_live_reference(port):
    import math
    rng = random.Random(20260923)
    for impl in O.ref_impls()[:2]:
        ref = O.Ref(impl)
        for _ in range(1500):
            body, _ = TF.string_body(rng, maxlen=rng.choice([80, 200]))
            assert port.parse_string(b'"' + body + b'"') == ref.parse_string(body + b'"'), body
        for _ in range(1500):
            tok = TF.scalar_token(rng)
            try:
                if not math.isfinite(float(tok.decode("latin1"))):
                    continue  # the reference rejects infinite VALUES (write_float); stage-2-lite does not convert floats
            except ValueError:
                pass
            doc, k = TF.wrap_scalar(tok, rng)
            r = port.stage1(doc)
            rerr, rtypes, rpay, _sb = ref.dom_tape(doc)
            if r.err != 0:
                assert rerr == r.err, doc
                continue
            err, types, pay, *_ = port.tokens(doc, r.idx, r.n)
            if rerr == 0:
                t, p = _tape_view(types, pay)
                assert err == 0 and t == bytes(rtypes), doc
                for i, ch in enumerate(t):
                    if chr(ch) in '"lu':
                        assert int(p[i]) == int(rpay[i]), doc
            else:
                assert types[k] == 0 and int(pay[k]) == rerr and err == rerr, (doc, err, int(pay[k]), rerr)
        for i in range(12):
            doc = bytes(corpus.random_json(rng.randrange(500, 60000), seed=777 + i))
            rerr, rtypes, rpay, rsb = ref.dom_tape(doc)
            keep = {str(j): int(rpay[j]) for j, t in enumerate(rtypes) if chr(t) in '"lu'}
            _check_doc_against(port, doc, rerr, bytes(rtypes), keep, bytes(rsb))
