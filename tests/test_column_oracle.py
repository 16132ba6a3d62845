"""The typed-column oracle (sjo_column, oracle/sj_column_oracle.c) pinned to the reference's DOM getters after
dom::element::at_pointer: for every document of tests/column_cases.py, the pointer corpora of tests/pointer_cases.py and
an array of 16 777 216 elements, and for get_int64, get_uint64, get_bool, get_string, get_array().size() and
get_object().size(), its error equals the reference's, and so do the value or the string's bytes on success.  Without the
reference, the same against tests/golden/columns.json."""
import json
import os

import pytest

import column_cases as CC
import column_oracle as CO
import oracle_lib as O
import pointer_cases as PC

GOLDEN = os.path.join(O.ROOT, "tests", "golden", "columns.json")


def check_against_reference(cols, ref, name, doc, pointers, kinds=CO.KINDS):
    for kind in kinds:
        _perr, want = ref.column(kind, doc, pointers)
        _tab, err, _rt, val, strs = cols.of_document(kind, doc, pointers)
        for p, (werr, wval, wbytes) in enumerate(want):
            assert err[p, 0] == werr, (name, kind, pointers[p], err[p, 0], werr)
            if werr == 0:
                got = strs[p] if kind == CO.STRING else int(val[p, 0])
                assert got == (wbytes if kind == CO.STRING else wval), (name, kind, pointers[p])


@pytest.mark.skipif(not CO.have_ref(), reason="reference build (oracle/_ref) not present")
def test_oracle_matches_reference():
    cols, ref = CO.Columns(), CO.RefColumns()
    for name, doc, pointers in CC.documents():
        check_against_reference(cols, ref, name, doc, pointers)
    for name, doc, pointers in PC.corpus_cases(full=False):
        if not name.startswith("bad"):
            check_against_reference(cols, ref, name, doc, pointers[:400])


@pytest.mark.skipif(not CO.have_ref(), reason="reference build (oracle/_ref) not present")
def test_size_saturates_like_the_reference():
    """the tape's scope count saturates at 0xFFFFFF: one past it, and exactly at it"""
    cols, ref = CO.Columns(), CO.RefColumns()
    for n in (0xFFFFFF, 0xFFFFFF + 1):
        doc = CC.big_array(n)
        check_against_reference(cols, ref, f"array{n}", doc, ["", "/0"], kinds=(CO.ARRAY_SIZE, CO.OBJECT_SIZE, CO.INT64))
        _tab, _err, _rt, val, _s = cols.of_document(CO.ARRAY_SIZE, doc, [""])
        assert int(val[0, 0]) == 0xFFFFFF


def test_oracle_matches_golden():
    g = json.load(open(GOLDEN))
    cols = CO.Columns()
    assert len(g["cases"]) >= 25
    for case in g["cases"]:
        doc = bytes.fromhex(case["doc"]) if "doc" in case else CC.document(case["name"])
        for kind_s, want in case["kinds"].items():
            kind = int(kind_s)
            _tab, err, _rt, val, strs = cols.of_document(kind, doc, case["pointers"])
            assert err[:, 0].tolist() == want["err"], (case["name"], kind)
            if kind == CO.STRING:
                assert [s.hex() for s in strs] == want["bytes"], (case["name"], kind)
            else:
                assert [str(int(v)) for v in val[:, 0]] == want["value"], (case["name"], kind)


def test_rows_that_select_no_value():
    """rows in error keep their error; an index past n, or at ',' ':' '}' ']', is UNEXPECTED_ERROR with row type 0"""
    cols = CO.Columns()
    port = O.Port()
    doc = b'{"a":[1,"x"],"b":true}'
    r = port.stage1(doc)
    tw = port.tokens(doc, r.idx, r.n)
    types = bytes(tw[1])
    rows_err = [20, 0, 0, 0, 0, 0, 0]
    rows_idx = [0xFFFFFFFF, r.n, types.index(b","), types.index(b":"), types.index(b"]"), types.index(b"}"), types.index(b'"', 3)]
    for kind in CO.KINDS:
        err, rt, val, _s = cols.column(kind, tw[1], tw[2], tw[3], len(tw[3]), rows_err, rows_idx)
        assert err.tolist()[:6] == [20, 24, 24, 24, 24, 24] and rt.tolist()[:6] == [0] * 6 and val.tolist()[:6] == [0] * 6
    # a string record outside [0, string_bytes): only STRING reads it
    err, rt, _v, _s = cols.column(CO.STRING, tw[1], tw[2], tw[3], 3, [0], [rows_idx[-1]])
    assert (err.tolist(), rt.tolist()) == ([24], [0])
    err, rt, _v, _s = cols.column(CO.INT64, tw[1], tw[2], tw[3], 3, [0], [rows_idx[-1]])
    assert (err.tolist(), rt.tolist()) == ([17], [ord('"')])
