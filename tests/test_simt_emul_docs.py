"""A multi-document launch of the scan4 kernel source under the host SIMT emulation (tests/simt_emul_docs.cpp): every
document's indexes, sentinels, carry and flags against the oracle, including a document boundary inside a look-back
window whose previous document ends inside a string.  No GPU involved."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    exe = str(tmp_path / "simt_emul_docs")
    inc = ["-I", os.path.join(ROOT, "simdjson_b200", "csrc"), "-I", os.path.join(ROOT, "oracle")]
    subprocess.check_call(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "sj_oracle.c"), "-o", str(tmp_path / "o.o")])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-pthread", *inc, os.path.join(ROOT, "tests", "simt_emul_docs.cpp"),
                           str(tmp_path / "o.o"), "-o", exe])
    return exe


def test_multi_document_launch_under_simt_emulation(tmp_path):
    out = subprocess.run([_build(tmp_path), "24"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    assert "simt emulation of multi-document launches OK" in out.stdout


def test_packed_documents_stay_inside_their_buffers(tmp_path):
    """documents packed back to back in one buffer (a neighbour ending in a backslash, an open string, a UTF-8 lead byte)
    and index arrays of exactly sjb200_index_words(len) words packed back to back in another, both against an
    inaccessible page: a read across a document's ends or a write outside its index array kills the process or shows"""
    out = subprocess.run([_build(tmp_path), "--fenced"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
    assert out.returncode == 0, (out.returncode, out.stdout[-2000:], out.stderr[-4000:])
    assert "simt emulation of packed, fenced multi-document launches OK" in out.stdout
