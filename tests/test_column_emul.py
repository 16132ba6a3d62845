"""CPU check of the size walk and the string copy of sjb200_column_dev (simdjson_b200/csrc/sjb200_column.cuh) under the
host SIMT emulation (tests/column_emul.cpp): the warp walk, the CTA walk and the hand-over from one to the other at the
warp's limit, against the oracle (sjo_column); group_copy at every source and destination phase and length around the
vector width, for a warp and a CTA.  The GPU run of the kernels is tests/test_column.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import column_cases as CC
import column_oracle as CO
import oracle_lib as O
import pointer_cases as PC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CTA_MIN = 4096  # SJB200_POINTER_CTA_MIN: the warp walk's limit


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("colemu") / "libcolemu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-I", os.path.join(ROOT, "simdjson_b200", "csrc"),
                           os.path.join(ROOT, "tests", "column_emul.cpp"), "-o", so])
    L = C.CDLL(so)
    L.emu_size.restype = C.c_longlong
    L.emu_size.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint64, C.POINTER(C.c_int)]
    L.emu_copy.restype = None
    L.emu_copy.argtypes = [C.c_uint, C.c_void_p, C.c_void_p, C.c_uint64]
    return L


def containers(doc):
    """tokens of doc and the structural indexes of its containers (at most 60, spread over the document)"""
    port = O.Port()
    r = port.stage1(doc)
    assert r.err == 0
    tw = port.tokens(doc, r.idx, r.n)
    ks = [k for k, t in enumerate(tw[1]) if t in (ord("["), ord("{"))]
    step = max(1, len(ks) // 60)
    return tw, ks[::step] + ks[:3]


def sizes(emu, tw, ks, warp_limit):
    types = np.ascontiguousarray(tw[1])
    out, handed = [], 0
    for k in ks:
        h = C.c_int(0)
        obj = int(types[k] == ord("{"))
        v = emu.emu_size(types.ctypes.data, len(types), k, obj, warp_limit, C.byref(h))
        assert v >= 0
        out.append(v)
        handed += h.value
    return out, handed


@pytest.mark.parametrize("warp_limit", [CTA_MIN, 64, 0], ids=["warp", "handover", "cta"])
def test_size_walk_matches_oracle(emu, warp_limit):
    cols = CO.Columns()
    docs = [CC.CONTAINERS] + [d for d, _p in CC.long_containers()] + [d for d, _p in PC.SMALL] + PC.random_docs(3, 5)
    handed_total = 0
    for doc in docs:
        tw, ks = containers(doc)
        if not ks:
            continue
        got, handed = sizes(emu, tw, ks, warp_limit)
        handed_total += handed
        for kind in (CO.ARRAY_SIZE, CO.OBJECT_SIZE):
            err, _rt, val, _s = cols.column(kind, tw[1], tw[2], tw[3], len(tw[3]), [0] * len(ks), ks)
            want = [int(v) for e, v in zip(err, val) if e == 0]
            mine = [g for g, e in zip(got, err) if e == 0]
            assert mine == want, (doc[:40], kind)
    if warp_limit == 64:
        assert handed_total >= 5  # the containers longer than one warp step


def test_size_walk_stops_at_n(emu):
    """an unclosed container is counted up to n, with no read past it"""
    types = np.frombuffer(b"[l,l,[l]", dtype=np.uint8).copy()
    h = C.c_int(0)
    for lim in (CTA_MIN, 2, 0):
        assert emu.emu_size(types.ctypes.data, len(types), 0, 0, lim, C.byref(h)) == 3


@pytest.mark.parametrize("width", [32, 256])
def test_group_copy(emu, width):
    rng = np.random.default_rng(11)
    src = rng.integers(0, 256, 4096 + 64, dtype=np.uint8)
    for so in range(16):
        for do in range(16):
            for n in list(range(0, 40)) + [63, 64, 65, 200, 1000, 4097]:
                dst = np.full(n + 64, 0xA5, dtype=np.uint8)
                emu.emu_copy(width, dst.ctypes.data + 16 + do, src.ctypes.data + so, n)
                assert bytes(dst[16 + do: 16 + do + n]) == bytes(src[so: so + n]), (so, do, n)
                assert (dst[: 16 + do] == 0xA5).all() and (dst[16 + do + n:] == 0xA5).all(), (so, do, n)
