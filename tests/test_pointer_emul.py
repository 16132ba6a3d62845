"""CPU check of the JSON Pointer walk (simdjson_b200/csrc/sjb200_pointer.cuh) and of its host compile of the pointers,
under the host SIMT emulation (tests/pointer_emul.cpp), for both group widths -- a warp, one structural per lane per step,
and a CTA of 8 warps, 8 structurals per thread per step -- against the oracle (sjo_at_pointer).  The GPU run of the
kernels is tests/test_at_pointer.py."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import pointer_oracle as PO
import pointer_cases as PC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ptremu") / "libptremu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-I", os.path.join(ROOT, "simdjson_b200", "csrc"),
                           os.path.join(ROOT, "tests", "pointer_emul.cpp"), "-o", so])
    L = C.CDLL(so)
    L.emu_at_pointer.restype = C.c_int
    L.emu_at_pointer.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_char_p, C.POINTER(C.c_size_t),
                                 C.c_int, C.c_void_p, C.c_void_p]
    return L


def run(L, cta, tw, pointers, root=0, end=None):
    types, pay, sb = tw[1], tw[2], tw[3]
    enc = [p.encode() for p in pointers]
    lens = (C.c_size_t * len(enc))(*[len(e) for e in enc])
    err = np.zeros(len(enc), dtype=np.int32)
    idx = np.zeros(len(enc), dtype=np.uint32)
    sb = sb if len(sb) else np.zeros(1, dtype=np.uint8)
    rc = L.emu_at_pointer(cta, types.ctypes.data, pay.ctypes.data, sb.ctypes.data, len(tw[3]), root, len(types) if end is None else end, b"".join(enc), lens,
                          len(enc), err.ctypes.data, idx.ctypes.data)
    assert rc == 0
    return err, idx


@pytest.mark.parametrize("cta", [0, 1], ids=["warp", "cta"])
def test_walk_matches_oracle(emu, cta):
    port = PO.Pointers()
    cases = [c for c in PC.corpus_cases(full=False) if not c[0].startswith("bad")]
    arr = json.dumps([{"i": i, "v": [i, str(i)]} if i % 3 else i for i in range(1500)]).encode()  # > one CTA step of structurals
    cases.append(("long", arr, ["", "/0", "/750/v/1", "/1499", "/1500", "/1498/i", "/-", "/x"]))
    for name, doc, pointers in cases:
        pointers = pointers[:25] + pointers[-15:] if len(pointers) > 40 else pointers  # paths first, mutations last
        _r, tw, _s, we, wi = port.table(doc, pointers)
        err, idx = run(emu, cta, tw, pointers)
        bad = [(pointers[p], int(err[p]), int(we[p, 0])) for p in range(len(pointers)) if err[p] != we[p, 0] or idx[p] != wi[p, 0]]
        assert not bad, (name, bad[:5])


def test_documents_of_a_stream(emu):
    """each row of an NDJSON stream walked within its own bounds"""
    port = PO.Pointers()
    doc = PC.stream_of(PC.amazon_rows(40))
    pointers = [f"/{i}" for i in range(10)] + ["/-", ""]
    r = port.port.stage1(doc)
    starts = PO.document_starts(doc, r.idx, r.n)
    _r, tw, _s, we, wi = port.table(doc, pointers, starts=starts)
    for d, s in enumerate(starts):
        end = starts[d + 1] if d + 1 < len(starts) else r.n
        err, idx = run(emu, 0, tw, pointers, s, end)
        assert err.tolist() == we[:, d].tolist() and idx.tolist() == wi[:, d].tolist()


def test_compile_limits(emu):
    tw = O.Port().tokens(b"[1]", np.array([0, 1, 2], dtype=np.uint32), 3)
    enc = ["/" + "/".join(["0"] * 1025)]
    lens = (C.c_size_t * 1)(len(enc[0]))
    e, i = np.zeros(1, dtype=np.int32), np.zeros(1, dtype=np.uint32)
    assert emu.emu_at_pointer(0, tw[1].ctypes.data, tw[2].ctypes.data, None, 0, 0, 3, enc[0].encode(), lens, 1, e.ctypes.data, i.ctypes.data) == 1
