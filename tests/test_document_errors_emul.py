"""CPU check of the stage-2 grammar pass (simdjson_b200/csrc/sjb200_grammar.cuh) under the host SIMT emulation
(tests/grammar_emul.cpp) against the oracle (sjo_document_errors).  Tiles of 32 and 64 structurals make small inputs
span many tiles: documents across many tiles and many documents per tile, errors on tile boundaries, stacks at the depth
cap across tiles, and broken documents followed by good ones.  The GPU run of the kernels is
tests/test_document_errors.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import grammar_oracle as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gramemu") / "libgramemu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-I", os.path.join(ROOT, "simdjson_b200", "csrc"),
                           os.path.join(ROOT, "tests", "grammar_emul.cpp"), "-o", so])
    L = C.CDLL(so)
    L.emu_document_errors.restype = C.c_int
    L.emu_document_errors.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def gram():
    return G.Grammar()


def check(L, g, doc, items, max_depth=1024, table=True):
    s = g.stream(doc, max_depth, table)
    assert s is not None
    _r, types, pay, starts, want_e, want_i = s
    D = len(starts) if starts else 1
    err = np.zeros(D, dtype=np.int32)
    idx = np.zeros(D, dtype=np.uint32)
    st = np.ascontiguousarray(starts if starts else [0], dtype=np.uint32)
    t = np.ascontiguousarray(types, dtype=np.uint8)
    p = np.ascontiguousarray(pay, dtype=np.uint64)
    assert L.emu_document_errors(items, t.ctypes.data, p.ctypes.data, len(t), st.ctypes.data if starts else None, D, max_depth, err.ctypes.data,
                                 idx.ctypes.data) == 0
    bad = [(d, int(err[d]), int(idx[d]), int(want_e[d]), int(want_i[d])) for d in range(D) if err[d] != want_e[d] or idx[d] != want_i[d]]
    assert not bad, (doc[:80], items, bad[:6])
    return err, idx


@pytest.mark.parametrize("items", [1, 2, 32])
def test_grammar_cases_one_at_a_time(emu, gram, items):
    for doc in G.grammar_cases() + G.stream_cases():
        if doc.strip() and gram.tokens(doc) is not None:
            check(emu, gram, doc, items, table=False)


@pytest.mark.parametrize("items", [1, 2])
def test_streams(emu, gram, items):
    cases = [c for c in G.grammar_cases() if c.strip()]
    check(emu, gram, b" ".join(cases), items)
    check(emu, gram, b"\n".join(cases), items)
    check(emu, gram, b"".join(G.stream_cases()), items)
    for doc in G.stream_cases():
        check(emu, gram, doc, items)


@pytest.mark.parametrize("items", [1, 2])
def test_depth_across_tiles(emu, gram, items):
    """stacks at the depth cap spanning tiles, empty containers at the limit, max_depth 1, 2, 3, 1024 and 4096"""
    for doc, md in G.depth_cases():
        if md <= 1024 or items == 2:
            check(emu, gram, doc, items, md, table=False)
    mixed = b"[" + b",".join(G.nested(d, b"1", "[{"[d % 2]) for d in range(1, 40)) + b"]"
    for md in (3, 17, 33, 64, 1024):
        check(emu, gram, mixed, items, md, table=False)
        check(emu, gram, b"\n".join([mixed, G.nested(70), mixed[:-1], mixed]), items, md)


@pytest.mark.parametrize("items", [1, 2, 32])
def test_fuzz(emu, gram, items):
    docs = G.fuzz_docs(300, seed=11 + items)
    check(emu, gram, b"\n".join(docs), items)
    check(emu, gram, b"".join(docs), items)
    for d in docs[:60]:
        check(emu, gram, d, items, table=False)


def test_broken_document_does_not_leak(emu, gram):
    """a document left open (its stack never popped) followed by good ones, each starting on a tile boundary or not"""
    good = b'{"a":[1,{"b":[2,3]},4],"c":{"d":null}}'
    for pad in range(0, 40, 3):
        for broken in (b"[" * 50 + b"1", b'{"x":[[[{"y":' + b"[" * 30 + b"2", b"[1,2" + b",[3" * 20):
            doc = b"[" + b"1," * pad + b"1]\n" + broken + b"\n" + b"\n".join([good] * 5)
            err, _ = check(emu, gram, doc, 1)
            assert err[0] == 0 and err[-1] == 0 and (err != 0).sum() >= 1
