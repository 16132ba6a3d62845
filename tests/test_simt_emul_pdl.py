"""Consecutive multi-document launches of the scan4 kernel source that overlap as programmatic dependent launch lets
them (tests/simt_emul_pdl.cpp), under the host SIMT emulation: index arrays shared by every launch, documents of one
element whose descriptors every launch starts at element 0, and a launch that reads what the previous one wrote.  No
GPU involved."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_overlapped_launches_under_simt_emulation(tmp_path):
    exe = str(tmp_path / "simt_emul_pdl")
    inc = ["-I", os.path.join(ROOT, "simdjson_b200", "csrc"), "-I", os.path.join(ROOT, "oracle")]
    subprocess.check_call(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "sj_oracle.c"), "-o", str(tmp_path / "o.o")])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-pthread", *inc, os.path.join(ROOT, "tests", "simt_emul_pdl.cpp"),
                           str(tmp_path / "o.o"), "-o", exe])
    out = subprocess.run([exe, "6"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    assert "simt emulation of overlapped launches OK" in out.stdout
