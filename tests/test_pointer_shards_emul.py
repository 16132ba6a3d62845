"""CPU check of the sharded JSON Pointer pass (sjb200_at_pointer_sharded): tests/pointer_shards_emul.cpp runs every rank's
walks (walk_from of sjb200_pointer.cuh with the rank's ShardCut) under the host SIMT emulation, warp and CTA groups, with
the pure edge fold (sjb200_fold.cpp) between the rounds and the continuation records carried from rank to rank.  1 to 8
ranks, every placement of one and two cuts in small documents, the pointer cases of tests/pointer_cases.py and seeded
random documents.  The gathered results must equal the oracle (sjo_at_pointer) on the whole stream and the unsharded
emulation (tests/pointer_emul.cpp).  The GPU run is tests/test_sharded_at_pointer.py."""
import ctypes as C
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

import pointer_cases as PC
import pointer_oracle as PO
from test_pointer_emul import emu, run  # noqa: F401  (the unsharded emulation, tests/pointer_emul.cpp)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "simdjson_b200", "csrc")
NONE64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def shards(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ptrshards") / "libptrshards.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-I", CSRC, os.path.join(ROOT, "tests", "pointer_shards_emul.cpp"),
                           os.path.join(CSRC, "sjb200_fold.cpp"), "-o", so])
    L = C.CDLL(so)
    L.emu_sharded_at_pointer.restype = C.c_int
    L.emu_sharded_at_pointer.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_uint32,
                                         C.c_char_p, C.POINTER(C.c_size_t), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def port():
    return PO.Pointers()


def _sharded(L, cta, tw, starts, whole, pointers, cuts):
    types, pay, sb = tw[1], tw[2], tw[3]
    N = len(types)
    # each rank's part of the string buffer starts at its first string's record
    sbase = []
    for r in range(len(cuts) - 1):
        q = [int(pay[k]) for k in range(cuts[r], N) if types[k] == ord('"')]
        sbase.append(q[0] if q else len(sb))
    sbase.append(len(sb))
    enc = [p.encode() for p in pointers]
    lens = (C.c_size_t * len(enc))(*[len(e) for e in enc])
    D = 1 if whole else len(starts)
    err = np.zeros((len(enc), max(D, 1)), dtype=np.int32)
    idx = np.zeros((len(enc), max(D, 1)), dtype=np.uint64)
    stats = np.zeros(3, dtype=np.uint64)
    t = np.ascontiguousarray(types, dtype=np.uint8) if N else np.zeros(1, np.uint8)
    p = np.ascontiguousarray(pay, dtype=np.uint64) if N else np.zeros(1, np.uint64)
    s = np.ascontiguousarray(sb, dtype=np.uint8) if len(sb) else np.zeros(1, np.uint8)
    c = np.ascontiguousarray(cuts, dtype=np.uint32)
    sbv = np.ascontiguousarray(sbase, dtype=np.uint64)
    st = np.ascontiguousarray(starts if starts else [0], dtype=np.uint32)
    rc = L.emu_sharded_at_pointer(cta, len(cuts) - 1, t.ctypes.data, p.ctypes.data, s.ctypes.data, c.ctypes.data, sbv.ctypes.data, int(whole), st.ctypes.data,
                                  0 if whole else len(starts), b"".join(enc), lens, len(enc), err.ctypes.data, idx.ctypes.data, stats.ctypes.data)
    assert rc == 0 and stats[2] == 0, (rc, stats)
    return err[:, :D], idx[:, :D], int(stats[0]), int(stats[1])


def _check(L, cta, tw, starts, whole, pointers, we, wi, cuts, what):
    err, idx, _rounds, _fw = _sharded(L, cta, tw, starts, whole, pointers, cuts)
    want_i = np.where(wi == 0xFFFFFFFF, np.uint64(NONE64), wi.astype(np.uint64))
    bad = [(pointers[p], d, int(err[p, d]), int(idx[p, d]), int(we[p, d]), int(want_i[p, d])) for p, d in zip(*np.nonzero((err != we) | (idx != want_i)))]
    assert not bad, (what, cuts, bad[:4])
    return _rounds, _fw


def nested_ok(types, s, e):
    """the brackets of structurals [s, e) match: where they do not, the walk deviates from the reference (documented)
    and the gathered call, not the oracle, is what the sharded pass must equal"""
    stack = []
    for t in types[s:e]:
        if t in (ord("{"), ord("[")):
            stack.append(t)
        elif t in (ord("}"), ord("]")):
            if not stack or stack.pop() != (ord("{") if t == ord("}") else ord("[")):
                return False
    return not stack


def _table(port, doc, pointers, whole):
    """(tokens, document starts, error[P, D], index[P, D]) of the gathered call: the unsharded emulation of the walk
    within each document, after the kernels' token-error rule; checked against the oracle where the nesting is valid"""
    r = port.port.stage1(doc)
    starts = None if whole else PO.document_starts(doc, r.idx, r.n)
    _r, tw, starts, we, wi = port.table(doc, pointers, starts=starts)
    types, pay = tw[1], tw[2]
    n = len(types)
    for d, s in enumerate(starts):
        end = starts[d + 1] if d + 1 < len(starts) else n
        bad = [k for k in range(s, end) if types[k] == 0]
        if bad:
            ue, ui = np.full(len(pointers), int(pay[bad[0]]) & 0xFF, np.int32), np.full(len(pointers), bad[0], np.uint32)
        else:
            ue, ui = run(emu_lib(), 0, tw, pointers, s, end)
        if nested_ok(types, s, end) or bad:
            assert ue.tolist() == we[:, d].tolist() and ui.tolist() == wi[:, d].tolist(), (doc, d)
        we[:, d], wi[:, d] = ue, ui
    return tw, ([] if whole else list(starts)), we, wi


CUT_DOCS = [
    (b'{"key": {"x": [10, 20, 30]}, "b": 1}', ["/key/x/2", "/key/x/3", "/key/y", "/b", "/key/x/0/z", "/b/0", "/key/x/1/q/r", "/-", "", "x", "/key/~2"]),
    (b'{"a": 1, "a": 2, "c": {"a": 3}}', ["/a", "/c/a", "/c/b", "/d", "/c/"]),
    (b'[[1, [2, [3, [4]]]], {"k": [[], {}]}, "s", 5]', ["/0/1/1/1/0", "/1/k/0", "/1/k/1/x", "/3", "/4", "/2/0", "/0/1/1/1/1", "/01"]),
    (b'{"a": {}} {"a": []} {"a": [1, 2]} [{"a": 1}] "x" {"a": {"b": 1}}', ["/a", "/a/0", "/a/1", "/a/b", "/0/a", ""]),
    (b'{"a": [1, tru, 3], "b": 2} {"b": [1, 2, 3]}', ["/b", "/a/0", "/b/2", "x"]),
    (b'{"a": [1, [2, 3}, "b": 2} {"b": {"c": ]]}', ["/b", "/a/1/1", "/b/c", "/a/1/5"]),  # nesting errors
    (b'{"a": 1 "b": 2} {"c": [3]}', ["/b", "/c/0"]),
    (b'[1] [2, [3', ["/0", "/1/0", "/1/1"]),
]


@pytest.mark.parametrize("cta", [0, 1], ids=["warp", "cta"])
def test_every_cut_of_small_documents(shards, port, cta):
    """every placement of one and two cuts: keys, colons and openers as a rank's last structural, arrays counted across
    cuts, duplicate keys on two ranks, errors decided on a later rank, ranks of 0, 1 and 2 structurals"""
    crossed = 0
    for doc, pointers in CUT_DOCS:
        for whole in (False, True):
            tw, starts, we, wi = _table(port, doc, pointers, whole)
            n = len(tw[1])
            for k in ((1, 2) if not cta else (1,)):  # (a CTA of OS threads is slow to start: one cut for it)
                for inner in itertools.combinations_with_replacement(range(n + 1), k):
                    crossed += _check(shards, cta, tw, starts, whole, pointers, we, wi, [0, *inner, n], (doc, whole))[1]
    assert crossed > 0


_EMU = []


def emu_lib():
    return _EMU[0]


@pytest.fixture(autouse=True)
def _keep_emu(emu):  # noqa: F811
    if not _EMU:
        _EMU.append(emu)


@pytest.mark.parametrize("cta", [0, 1], ids=["warp", "cta"])
def test_pointer_cases_across_ranks(shards, port, cta):
    """the pointer cases (every path and its mutations) of the small corpus documents, one document across 2 to 8 ranks"""
    rng = random.Random(300 + cta)
    cases = [c for c in PC.corpus_cases(full=False) if c[0] not in ("twitter", "citm")][:8]
    for name, doc, pointers in cases:
        pointers = pointers[:20] + pointers[-10:] if len(pointers) > 30 else pointers
        tw, starts, we, wi = _table(port, doc, pointers, True)
        n = len(tw[1])
        for world in (2, 3, 4, 8):
            cuts = [0] + sorted(rng.randrange(0, n + 1) for _ in range(world - 1)) + [n]
            _check(shards, cta, tw, starts, True, pointers, we, wi, cuts, name)


def test_random_documents_as_a_stream(shards, port):
    """seeded random documents as one whitespace-separated stream, 1 to 8 ranks, warp and CTA groups"""
    rng = random.Random(301)
    docs = PC.random_docs(12, seed=5)
    stream = b"\n".join(docs)
    pointers = ["", "/0", "/1", "/a", "/0/0", "/-", "/x/y"]
    for d in docs[:3]:
        try:
            import json
            v = json.loads(d)
            pointers += list(PC.paths(v, 3))[:15]
        except ValueError:
            pass
    tw, starts, we, wi = _table(port, stream, pointers, False)
    n = len(tw[1])
    for world in range(1, 9):
        for cta in (0, 1):
            cuts = [0] + sorted(rng.randrange(0, n + 1) for _ in range(world - 1)) + [n]
            _check(shards, cta, tw, starts, False, pointers, we, wi, cuts, ("random", world))


def test_whole_document_targets_on_every_rank(shards, port):
    import json
    doc = json.dumps([{"i": i, "v": [i, str(i), {"d": [[i]]}]} for i in range(300)]).encode()
    pointers = ["/0", "/150/v/2/d/0/0", "/299", "/299/v/1", "/300", "/-", "/1/x", ""]
    tw, starts, we, wi = _table(port, doc, pointers, True)
    n = len(tw[1])
    for world in (2, 3, 4, 8):
        cuts = [n * k // world for k in range(world + 1)]
        for cta in (0, 1):
            rounds, fw = _check(shards, cta, tw, starts, True, pointers, we, wi, cuts, world)
            assert rounds == world - 1 and fw > 0
