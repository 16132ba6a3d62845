"""CPU check of get_double in sjb200_column_double_dev (simdjson_b200/csrc/sjb200_double.cuh): the host build of the
device routine -- the lane's summary, the Clinger and Eisel-Lemire paths and the exact comparison -- against Python's
float() (correctly rounded) bit for bit, on the named cases and on 2 M seeded numbers; the long-number summary by a warp
and by a CTA under the host SIMT emulation (tests/double_emul.cpp); and the committed power-of-five table against its
generator.  The GPU run of the kernels is tests/test_column_double.py."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import double_cases as DC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("dblemu") / "libdblemu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-ffp-contract=off", "-I",
                           os.path.join(ROOT, "simdjson_b200", "csrc"), os.path.join(ROOT, "tests", "double_emul.cpp"), "-o", so])
    L = C.CDLL(so)
    L.emu_double_lane.restype = None
    L.emu_double_lane.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_double_group.restype = C.c_int
    L.emu_double_group.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    return L


def lane(emu, texts):
    enc = [t.encode() for t in texts]
    buf = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    offs = np.zeros(len(enc) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(t) for t in enc])
    err = np.zeros(len(enc), dtype=np.int32)
    bits = np.zeros(len(enc), dtype=np.uint64)
    slow = np.zeros(len(enc), dtype=np.int32)
    emu.emu_double_lane(buf.ctypes.data, offs.ctypes.data, len(enc), err.ctypes.data, bits.ctypes.data, slow.ctypes.data)
    return err, bits, slow


def check_lane(emu, texts):
    err, bits, slow = lane(emu, texts)
    want = [DC.expect(t, as_token=False) for t in texts]
    we = np.array([w[0] for w in want], dtype=np.int32)
    wb = np.array([w[1] for w in want], dtype=np.uint64)
    bad = np.flatnonzero((err != we) | (bits != wb))
    assert len(bad) == 0, [(texts[i][:60], int(err[i]), hex(int(bits[i])), int(we[i]), hex(int(wb[i]))) for i in bad[:5]]
    return slow


def test_named_cases(emu):
    slow = check_lane(emu, DC.named_cases())
    assert slow.sum() >= 20  # the halfway points and the long tails take the exact comparison


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_random_numbers(emu, seed):
    """2 M numbers over the four seeds"""
    check_lane(emu, DC.random_numbers(500_000, seed))


def test_slow_heavy(emu):
    check_lane(emu, DC.slow_heavy(20000, 7))


def test_not_a_number(emu):
    """a span that is not a JSON number (a corrupted payload) is UNEXPECTED_ERROR, never read past"""
    texts = ["", "-", "+1", "1.", ".5", "1e", "1e+", "01", "1.2.3", "1e5e5", "1-2", "--1", "1x", "e5", "0x10", "1 ", "-.5", "1E+-5"]
    err, bits, _slow = lane(emu, texts)
    assert err.tolist() == [24] * len(texts) and bits.tolist() == [0] * len(texts)


@pytest.mark.parametrize("cta", [0, 1], ids=["warp", "cta"])
def test_group_summary(emu, cta):
    """long numbers summarized by a warp and by a CTA, converted as dbl_long_kernel does"""
    big = "1" + "0" * 70000 + "e-70000"
    texts = DC.named_cases() + DC.long_tail(3000) + [big, "0." + "0" * 5000 + "1234e5010", "1" + "0" * 400 + ".5e-390", "-" + "9" * 1000,
                                                      "1e" + "0" * 3000 + "5", "0." + "1" * 900, "1.5e-" + "0" * 40 + "1"]
    for t in texts:
        b = C.c_uint64()
        s = C.c_int32()
        e = emu.emu_double_group(t.encode(), len(t), cta, C.byref(b), C.byref(s))
        want = DC.expect(t, as_token=False)
        assert (e, b.value) == want, (t[:50], len(t), e, hex(b.value), want)


def test_pow5_table_matches_generator():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_pow5
    with open(os.path.join(ROOT, "simdjson_b200", "csrc", "sjb200_pow5.h")) as f:
        assert f.read() == gen_pow5.header()
    for q in (-342, -27, -1, 0, 1, 27, 55, 308):
        T, t = gen_pow5.entry(q)
        exact = 5 ** q if q >= 0 else None
        if exact is not None:
            assert T == (exact >> t if t >= 0 else exact << -t)
        else:
            assert T * 5 ** -q <= 2 ** -t < (T + 1) * 5 ** -q
