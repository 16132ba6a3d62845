"""A multi-document launch of the scan4 kernel source under the host SIMT emulation (tests/simt_emul_docs.cpp): every
document's indexes, sentinels, carry and flags against the oracle, including a document boundary inside a look-back
window whose previous document ends inside a string.  No GPU involved."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_multi_document_launch_under_simt_emulation(tmp_path):
    exe = str(tmp_path / "simt_emul_docs")
    inc = ["-I", os.path.join(ROOT, "simdjson_b200", "csrc"), "-I", os.path.join(ROOT, "oracle")]
    subprocess.check_call(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "sj_oracle.c"), "-o", str(tmp_path / "o.o")])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-pthread", *inc, os.path.join(ROOT, "tests", "simt_emul_docs.cpp"),
                           str(tmp_path / "o.o"), "-o", exe])
    out = subprocess.run([exe, "24"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    assert "simt emulation of multi-document launches OK" in out.stdout
