"""The scan4 kernel SOURCE (simdjson_b200/csrc/sjb200_scan4.cuh), compiled for the host SIMT emulation and run against
the oracle: one OS thread per CUDA thread, warp collectives as rendezvous, mbarriers with deferred TMA copies
(sjb200_simt.cuh, SJB200_HOST_EMU).  Covers the warp roles, the ticket / mbarrier pipeline, the both-polarity block
scans, the look-back chain (several CTAs, windows), emit, launch carries, chunked launches, shard transducers, plain-load
and misaligned paths, minify on the scan4 structure.  (Built with -fsanitize=thread the same program reports no data
race in the shared-memory / mbarrier protocol; that build is too slow for the regular run.)  No GPU involved; the GPU parity tests live in test_gpu_parity.py."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    exe = str(tmp_path / "simt_emul")
    inc = ["-I", os.path.join(ROOT, "simdjson_b200", "csrc"), "-I", os.path.join(ROOT, "oracle")]
    subprocess.check_call(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "sj_oracle.c"), "-o", str(tmp_path / "o.o")])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-pthread", *inc, os.path.join(ROOT, "tests", "simt_emul.cpp"),
                           str(tmp_path / "o.o"), "-o", exe])
    return exe


def test_scan4_kernel_source_under_simt_emulation(tmp_path):
    out = subprocess.run([_build(tmp_path), "140"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    assert "simt emulation OK" in out.stdout


def test_scan4_and_utf8v2_stay_inside_their_buffers(tmp_path):
    """stage 1 (every incoming shard state), minify and utf8v2 with the input ending exactly at, or starting right after, an
    inaccessible page, and the index output (sjb200_index_words(len) words) and the minify destination (len bytes) against
    one too, TMA on and off, at lengths around 128, 4096 and the tile: an access outside a buffer kills the process"""
    out = subprocess.run([_build(tmp_path), "--fenced"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
    assert out.returncode == 0, (out.returncode, out.stdout[-2000:], out.stderr[-4000:])
    assert "simt emulation, fenced buffers OK" in out.stdout
