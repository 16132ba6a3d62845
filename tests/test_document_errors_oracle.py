"""The grammar oracle (oracle/sj_grammar_oracle.c, sjo_document_errors) pinned against the live reference's stage 2
(skipped without it) and against tests/golden/document_errors.json.  Error codes are pinned against the reference; the
indexes of errors against the oracle only, because the reference does not expose them.  The documented deviations are
asserted as such: a root token that starts with a byte below '0' other than '-', a float whose value is infinite, and
the last document of a stream that wants a value past the end."""
import numpy as np
import pytest

import grammar_oracle as G


@pytest.fixture(scope="module")
def gram():
    return G.Grammar()


@pytest.fixture(scope="module")
def ref():
    if not G.have_ref():
        pytest.skip("reference not built (oracle/grammar.mk)")
    return G.RefGrammar()


def pin_whole(g, ref, doc, max_depth=1024):
    s = g.stream(doc, max_depth, table=False)
    if s is None:
        return None
    r, _t, _p, _s, err, idx = s
    want = ref.parse(doc, max_depth) if r.n else G.EMPTY
    assert G.agrees(doc, r, None, 0, int(err[0]), int(idx[0]), want, None), (doc[:80], int(err[0]), int(idx[0]), want)
    return int(err[0]), int(idx[0])


def pin_stream(g, ref, doc, max_depth=1024):
    s = g.stream(doc, max_depth)
    if s is None:
        return None
    r, _t, _p, starts, err, idx = s
    _e1, re_, rn, _n = ref.stream(doc, starts, max_depth)
    for d in range(len(starts)):
        we, wi = G.expected_from_ref(re_[d], rn[d], starts, d, r.n)
        assert G.agrees(doc, r, starts, d, int(err[d]), int(idx[d]), we, wi), (doc[:80], d, int(err[d]), int(idx[d]), we, wi)
    return err, idx


def test_every_return_and_token_error(gram, ref):
    n = 0
    for doc in G.grammar_cases() + G.stream_cases():
        n += pin_whole(gram, ref, doc) is not None
    assert n > 150


def test_indexes(gram):
    """where each error is decided, from the walk's own definition"""
    cases = {b'[1 2]': (3, 2), b'{"a" 1}': (3, 2), b'[1,]': (3, 3), b'[,1]': (9, 1), b'[1]]': (3, 3), b'1 2': (3, 1), b'[1,2': (3, 0),
             b'{"a":tru}': (6, 3), b'{tru:1}': (3, 1), b'{"\\x":1}': (5, 1), b'[[]': (3, 3), b'"a"': (0, 1), b'[]': (0, 2),
             b'[1 tru]': (3, 2), b'+1': (9, 0)}
    for doc, want in cases.items():
        s = gram.stream(doc, table=False)
        assert (int(s[4][0]), int(s[5][0])) == want, doc
    s = gram.stream(b'[1] [2')  # the last document wants a value past n
    assert s[4].tolist() == [0, 3] and s[5].tolist() == [3, 5]
    s = gram.stream(b'[1,2] [3 4] [5]')  # `4 ]` is cut as its own document: the walk ends before its end
    assert s[4].tolist() == [0, 3, 3, 0] and s[5][2] == 8


def test_depth(gram, ref):
    for doc, md in G.depth_cases():
        pin_whole(gram, ref, doc, md)
    assert pin_whole(gram, ref, G.nested(3, b"[]"), 4) == (0, 8)
    assert pin_whole(gram, ref, G.nested(4), 4) == (G.DEPTH_ERROR, 3)


def test_streams(gram, ref):
    for doc in G.stream_cases():
        pin_stream(gram, ref, doc)
    cases = [c for c in G.grammar_cases() if c.strip()]
    pin_stream(gram, ref, b" ".join(cases))
    pin_stream(gram, ref, b"\n".join(cases))


def test_root_scalars_glued_and_at_the_end(gram, ref):
    for doc in (b'1"a"', b'true"x"', b'false[1]', b'null{}', b'-1"b"', b'1.5e3"c"', b'"a"1', b'12', b'true', b'"x"'):
        pin_whole(gram, ref, doc)
        pin_stream(gram, ref, doc)
    assert gram.errors(np.zeros(0, dtype=np.uint8), np.zeros(0, dtype=np.uint64))[0].tolist() == [G.EMPTY]


def test_deviations(gram, ref):
    # a float whose value is infinite: grammar only here
    s = gram.stream(b"[1e400]", table=False)
    assert s[4][0] == 0 and ref.parse(b"[1e400]") == G.NUMBER_ERROR
    # a root token below '0' other than '-': judged as inside a container here
    for doc in (b"+1", b"#", b".5"):
        assert gram.stream(doc, table=False)[4][0] == G.NUMBER_ERROR and ref.parse(doc) == G.TAPE_ERROR
        assert ref.parse(b"[" + doc + b"]") == G.NUMBER_ERROR


def test_mutation_fuzz(gram, ref):
    docs = G.fuzz_docs(3000)
    bad = sum(pin_whole(gram, ref, d)[0] != 0 for d in docs)
    assert bad > 1000
    err, _ = pin_stream(gram, ref, b"\n".join(docs))
    assert (err != 0).sum() > 500
    pin_stream(gram, ref, b"".join(docs))


def test_golden(gram):
    gold = G.load_golden()
    assert len(gold["cases"]) > 300
    for case in gold["cases"]:
        doc = bytes.fromhex(case["doc"])
        s = gram.stream(doc, case["max_depth"], table=case["stream"])
        assert s[4].tolist() == case["errors"] and s[5].tolist() == case["indexes"], doc[:80]


def test_bad_tables(gram):
    types = np.frombuffer(b"[l]", dtype=np.uint8)
    pay = np.zeros(3, dtype=np.uint64)
    for starts in ([0, 0], [0, 3], [1, 0]):
        e, i = gram.errors(types, pay, starts)
        assert e.tolist() == [24, 24] and i.tolist() == [G.NONE] * 2
