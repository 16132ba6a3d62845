"""CPU check of the sharded stage-2 grammar (sjb200_document_errors_sharded): tests/grammar_shards_emul.cpp runs every
rank's share of the kernels' tile routines (sjb200_grammar.cuh, with the rank's ShardHalo) under the host SIMT
emulation, and the pure host folds (sjb200_fold.cpp) between the rounds.  1 / 2 / 4 / 8 ranks, tiles of 32, 64 and
1 024 structurals, cuts at token positions on, next to and inside tiles -- including ranks with 0, 1 and 2 structurals
-- and every cut of small documents.  The gathered results and the summary must equal the oracle (sjo_document_errors)
on the whole stream and the unsharded emulation (tests/grammar_emul.cpp).  The GPU run is
tests/test_sharded_document_errors.py."""
import ctypes as C
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

import grammar_oracle as G
from test_document_errors_emul import emu  # noqa: F401  (the unsharded emulation, tests/grammar_emul.cpp)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "simdjson_b200", "csrc")
NONE64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def shards(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gramshards") / "libgramshards.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-I", CSRC, os.path.join(ROOT, "tests", "grammar_shards_emul.cpp"),
                           os.path.join(CSRC, "sjb200_fold.cpp"), "-o", so])
    L = C.CDLL(so)
    L.emu_sharded_document_errors.restype = C.c_int
    L.emu_sharded_document_errors.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_uint32,
                                              C.c_void_p, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def gram():
    return G.Grammar()


def _sharded(L, items, types, pay, cuts, starts, whole, md):
    D = 1 if whole else len(starts)
    err = np.full(max(D, 1), -1, dtype=np.int32)
    idx = np.zeros(max(D, 1), dtype=np.uint64)
    summ = np.zeros(6, dtype=np.uint64)
    t = np.ascontiguousarray(types, dtype=np.uint8) if len(types) else np.zeros(1, np.uint8)
    p = np.ascontiguousarray(pay, dtype=np.uint64) if len(types) else np.zeros(1, np.uint64)
    c = np.ascontiguousarray(cuts, dtype=np.uint32)
    st = np.ascontiguousarray(starts if starts else [0], dtype=np.uint32)
    assert L.emu_sharded_document_errors(items, len(cuts) - 1, t.ctypes.data, p.ctypes.data, c.ctypes.data, int(whole), st.ctypes.data,
                                         0 if whole else len(starts), md, err.ctypes.data, idx.ctypes.data, summ.ctypes.data) == 0
    return err[:D], idx[:D], [int(x) for x in summ]


def _check(L, U, items, types, pay, starts, want_e, want_i, cuts, whole, md, what):
    err, idx, summ = _sharded(L, items, types, pay, cuts, starts, whole, md)
    if not whole and not starts:
        assert summ[:3] == [0, 0, 0], what
        return
    wi = np.where(np.asarray(want_i) == 0xFFFFFFFF, np.uint64(NONE64), np.asarray(want_i, dtype=np.uint64))
    bad = [(d, int(err[d]), int(idx[d]), int(want_e[d]), int(wi[d])) for d in range(len(want_e)) if err[d] != want_e[d] or idx[d] != wi[d]]
    assert not bad, (what, cuts, bad[:4])
    nerr = int((np.asarray(want_e) != 0).sum())
    fd = int(np.argmax(np.asarray(want_e) != 0)) if nerr else NONE64
    assert summ[0] == 0 and summ[1] == len(want_e) and summ[2] == nerr and summ[3] == fd, (what, cuts, summ)
    if nerr:
        assert (summ[4], summ[5]) == (int(want_e[fd]), int(wi[fd])), (what, cuts, summ)
    if len(types) and U is not None:  # the unsharded emulation on the same tokens
        D = len(want_e)
        ue, ui = np.zeros(D, np.int32), np.zeros(D, np.uint32)
        st = np.ascontiguousarray(starts if starts else [0], dtype=np.uint32)
        t, p = np.ascontiguousarray(types, dtype=np.uint8), np.ascontiguousarray(pay, dtype=np.uint64)
        assert U.emu_document_errors(items, t.ctypes.data, p.ctypes.data, len(t), None if whole else st.ctypes.data, D, md, ue.ctypes.data,
                                     ui.ctypes.data) == 0
        assert np.array_equal(ue, err) and np.array_equal(ui.astype(np.uint64), idx), (what, cuts)


def _cut_sets(n, world, tile, rng, count):
    """token cuts: on, next to and inside tiles, and random ones (empty ranks included)"""
    near = sorted({x for k in range(0, n + 1, tile) for x in (k - 1, k, k + 1) if 0 <= x <= n})
    for _ in range(count):
        pool = near if rng.random() < 0.5 else range(n + 1)
        inner = sorted(rng.choice(pool) for _ in range(world - 1))
        yield [0] + inner + [n]


def _stream(gram, doc, md=1024, table=True):
    s = gram.stream(doc, md, table)
    assert s is not None
    _r, types, pay, starts, e, i = s
    return types, pay, (list(starts) if starts else []), e, i


@pytest.mark.parametrize("items", [1, 2, 32])
def test_golden_cases_as_a_stream(shards, emu, gram, items):  # noqa: F811
    rng = random.Random(100 + items)
    gold = [bytes.fromhex(c["doc"]) for c in G.load_golden()["cases"] if c["max_depth"] == 1024 and c["doc"]]
    for sep in ((b"\n", b" ") if items == 32 else (b"\n",)):
        types, pay, starts, e, i = _stream(gram, sep.join(gold))
        for world in (1, 2, 4, 8):
            for cuts in _cut_sets(len(types), world, 32 * items, rng, 6 if items == 32 else 2):
                _check(shards, emu, items, types, pay, starts, e, i, cuts, False, 1024, ("golden", sep, world))


@pytest.mark.parametrize("items", [1, 2, 32])
def test_fuzz_set(shards, emu, gram, items):  # noqa: F811
    rng = random.Random(200 + items)
    docs = G.fuzz_docs(200 if items == 32 else 80, seed=31 + items)
    types, pay, starts, e, i = _stream(gram, b"\n".join(docs))
    for world in (2, 4, 8):
        for cuts in _cut_sets(len(types), world, 32 * items, rng, 6):
            _check(shards, emu, items, types, pay, starts, e, i, cuts, False, 1024, ("fuzz", world))
    for d in docs[:40]:  # one document across ranks
        types, pay, _, e, i = _stream(gram, d, table=False)
        for world in (2, 4):
            for cuts in _cut_sets(len(types), world, 32 * items, rng, 2):
                _check(shards, emu, items, types, pay, [], e, i, cuts, True, 1024, ("fuzz whole", d[:40], world))


CUT_DOCS = [
    b'{"a": 1 "b": 2}\n{"c": 3}', b'[1, 2] ] [3]', b'{"key": 1, "k2": 2}', b'[[]]', b'{"a": {}, "b": []}', b'[1] [2] [3]', b'[1] [2, [3',
    b'[1]', b'[1, 2]', b'{"a": [1, 2]}', b'1 2 3', b'[1,]', b'[{}]', b'{"a":1,}', b'[1]]', b'] [1]', b'{"a" 1}', b'[1 tru] 2',
]


@pytest.mark.parametrize("items", [1, 32])
def test_every_cut_of_small_documents(shards, emu, gram, items):  # noqa: F811
    """every placement of one and two cuts: each cut at a first or last structural of a shard, ranks of 0 / 1 / 2"""
    for doc in CUT_DOCS + [c for c in G.grammar_cases() if c.strip()][::29]:
        for whole in (False, True):
            s = gram.stream(doc, 1024, not whole)
            if s is None:
                continue
            _r, types, pay, starts, e, i = s
            starts = list(starts) if starts else []
            n = len(types)
            for k in (1, 2):
                for inner in itertools.combinations_with_replacement(range(n + 1), k):
                    _check(shards, emu, items, types, pay, starts, e, i, [0, *inner, n], whole, 1024, (doc, whole))


@pytest.mark.parametrize("items", [1, 2])
def test_depth_limit_at_the_cut(shards, emu, gram, items):  # noqa: F811
    """max_depth 1, 2, 3, 31, 32, 33, 1024, 4096 reached at, before and after the cut; empty pairs at the limit split by it"""
    for md in (1, 2, 3, 31, 32, 33, 1024, 4096):
        for depth in (md - 1, md, md + 1):
            if depth < 1:
                continue
            for inner in (b"1", b"[]"):
                for kind in ("[{" if md <= 33 else "["):
                    doc = G.nested(depth, inner, kind)
                    for whole, d in ((True, doc), (False, b"[1]\n" + doc + b"\n[2]")):
                        s = gram.stream(d, md, not whole)
                        _r, types, pay, starts, e, i = s
                        starts = list(starts) if starts else []
                        n = len(types)
                        at = d.count(b"[", 0, d.index(inner)) + d.count(b"{", 0, d.index(inner)) + d.count(b":", 0, d.index(inner))
                        for c in {at - 1, at, at + 1}:
                            if 0 <= c <= n:
                                _check(shards, emu, items, types, pay, starts, e, i, [0, c, n], whole, md, (md, depth, inner, kind, whole, c))
