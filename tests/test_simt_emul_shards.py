"""The per-shard launches of sharded minify / validate_utf8 / stage 1 from the kernel sources under the host SIMT emulation
(tests/simt_emul_shards.cpp), exchange windows in host memory: every record (seq, kind, count, state, transducer, flags)
against the oracle, re-minified shards with a non-zero carry-in against the oracle's minify of the whole buffer, and
utf8v2's record for valid and corrupted shards.  No GPU involved."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_minify_utf8_records_under_simt_emulation(tmp_path):
    exe = str(tmp_path / "simt_emul_shards")
    inc = ["-I", os.path.join(ROOT, "simdjson_b200", "csrc"), "-I", os.path.join(ROOT, "oracle")]
    subprocess.check_call(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "sj_oracle.c"), "-o", str(tmp_path / "o.o")])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-pthread", *inc, os.path.join(ROOT, "tests", "simt_emul_shards.cpp"),
                           str(tmp_path / "o.o"), "-o", exe])
    out = subprocess.run([exe, "6"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    assert "simt emulation of sharded minify / validate_utf8 records OK" in out.stdout
