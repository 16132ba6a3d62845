"""The JSON Pointer oracle (sjo_at_pointer, oracle/sj_pointer_oracle.c) pinned to the reference's dom::element::at_pointer: on
twitter, citm, escaped / empty / duplicate keys, bad tokens and seeded random documents, its error equals the
reference's, and on success the raw span it names, parsed and minified by the reference, equals the reference's
serialisation of the element.  Without the reference, the same against tests/golden/pointers.json."""
import json
import os

import pytest

import oracle_lib as O
import pointer_oracle as PO
import pointer_cases as PC

GOLDEN = os.path.join(O.ROOT, "tests", "golden", "pointers.json")


def oracle_results(port, doc, pointers):
    r, tw, _starts, err, idx = port.table(doc, pointers)
    assert r.err == 0
    return r, tw, err[:, 0], idx[:, 0]


@pytest.mark.skipif(not PO.have_ref(), reason="reference build (oracle/_ref) not present")
def test_oracle_matches_reference():
    port, ref, rp = PO.Pointers(), O.Ref(), PO.RefPointers()
    checked = 0
    for name, doc, pointers in PC.corpus_cases(full=True):
        r, tw, err, idx = oracle_results(port, doc, pointers)
        want = rp.at_pointer(doc, pointers)
        for p, ptr in enumerate(pointers):
            werr, wval = want[p]
            assert err[p] == werr, (name, ptr, err[p], werr)
            if werr == 0:
                span = PO.value_span(doc, r.idx, tw[1], idx[p])
                rerr, got = ref.dom_roundtrip(span)
                assert rerr == 0 and got == wval, (name, ptr, span[:80], wval[:80])
            checked += 1
    assert checked > 20000


@pytest.mark.skipif(not PO.have_ref(), reason="reference build (oracle/_ref) not present")
def test_oracle_matches_reference_on_rows():
    """amazon rows (arrays, /0 to /9) and twitter statuses (objects), each row a document"""
    port, ref, rp = PO.Pointers(), O.Ref(), PO.RefPointers()
    rows = [(r, [f"/{i}" for i in range(11)] + ["/-", ""]) for r in PC.amazon_rows(60)]
    rows += [(r, ["/id", "/user/id", "/user/screen_name", "/entities/hashtags/0/text", "/retweeted_status/user/id", "/text", "/x"])
             for r in PC.twitter_rows()]
    for doc, pointers in rows:
        r, tw, err, idx = oracle_results(port, doc, pointers)
        for p, (werr, wval) in enumerate(rp.at_pointer(doc, pointers)):
            assert err[p] == werr, (doc[:60], pointers[p])
            if werr == 0:
                assert ref.dom_roundtrip(PO.value_span(doc, r.idx, tw[1], idx[p]))[1] == wval


def test_oracle_matches_golden():
    g = json.load(open(GOLDEN))
    port = PO.Pointers()
    for case in g["cases"]:
        doc = O.jsonexample(case["file"]) if "file" in case else bytes.fromhex(case["doc"])
        r, _tw, err, idx = oracle_results(port, doc, case["pointers"])
        assert err.tolist() == case["err"], case.get("file", case["doc"][:40])
        got = [int(r.idx[k]) if e == 0 else -1 for e, k in zip(err, idx)]
        assert got == case["byte"], case.get("file", case["doc"][:40])


def test_token_error_wins():
    """a document with a bad number or atom answers every pointer with its first token in error"""
    port = PO.Pointers()
    for doc in PC.BAD:
        r = port.port.stage1(doc)
        tw = port.port.tokens(doc, r.idx, r.n)
        assert tw[0] != 0
        for ptr in ("", "/a", "/0", "/zz/1", "x"):
            assert port.at_pointer(tw[1], tw[2], tw[3], ptr) == (tw[0], tw[6])
