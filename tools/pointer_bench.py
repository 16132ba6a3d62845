"""JSON Pointer lookup on the device (sjb200_at_pointer_dev), timed next to the stage-1, document-table and tokens calls
of the same input.  Inputs:
  twitter_1g  1 GiB of NDJSON rows, the statuses of twitter.json repeated; four pointers per row
  doc_64m     the 64 MiB corpus.random_json document; pointers to its first, middle and last root elements
Every time is the median over --calls calls, CUDA events around the call (each call ends in its own synchronise).
Outputs are checked against the oracle (sjo_at_pointer) on the same bytes: a seeded sample of rows, the whole document.
Prints the GPU's name, power limit and SM clock, then one JSON line per input.

--sweep L1,L2,..: the warp walk against the CTA walk on streams of documents of about L structurals each (~4 M
structurals per stream, the last element of each looked up), for choosing SJB200_POINTER_CTA_MIN.  It loads the two
builds of tools/build_variants.sh  warp "-DSJB200_POINTER_CTA_MIN=0xFFFFFFFF" cta "-DSJB200_POINTER_CTA_MIN=0".

    python tools/pointer_bench.py [--calls 10] [--inputs twitter_1g,doc_64m] [--sweep 64,256,1024,4096,16384,65536]
"""
import argparse
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pointer_oracle as PO  # noqa: E402
import pointer_cases as PC  # noqa: E402
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import capi, corpus  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except (OSError, subprocess.SubprocessError, IndexError):
        return {"name": torch.cuda.get_device_name(), "note": "nvidia-smi not available"}


def timed(fn, calls):
    """median ms over `calls` calls after one warm-up, CUDA events around each"""
    fn()
    ms = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), ms


class Input:
    """one input resident in HBM with stage 1, the document table and the tokens computed once"""

    def __init__(self, doc):
        self.doc = doc
        self.d = torch.from_numpy(np.frombuffer(doc, dtype=np.uint8).copy()).cuda()
        rc, self.p = sj.get_active_implementation().create_dom_parser_implementation(len(doc))
        assert rc == sj.SUCCESS
        self.stage1()
        self.n = self.p.n_structural_indexes
        self.d_idx = self.p.device_index_buffer()
        self.table = torch.empty(2 * (self.n + 1), dtype=torch.int32, device="cuda")
        self.ndocs = self.doc_table()
        self.cap = int(sj.lib().sjb200_string_buf_capacity(len(doc)))
        self.d_type = torch.empty(max(self.n, 1), dtype=torch.uint8, device="cuda")
        self.d_payload = torch.empty(max(self.n, 1), dtype=torch.int64, device="cuda")
        self.d_strbuf = torch.empty(self.cap, dtype=torch.uint8, device="cuda")
        self.res = capi.TokensResult()
        assert self.tokens() == 0, self.res.error

    def stage1(self):
        assert self.p.stage1_device(self.d, sj.REGULAR) == sj.SUCCESS

    def doc_table(self):
        nd = C.c_uint32(0)
        assert sj.lib().sjb200_document_table_dev(self.p._ctx, self.d.data_ptr(), self.p.device_index_buffer().data_ptr(), self.n, self.table.data_ptr(),
                                                  self.n + 1, C.byref(nd), None) == 0
        return nd.value

    def tokens(self):
        return sj.lib().sjb200_tokens_dev(self.p._ctx, self.d.data_ptr(), self.d.numel(), self.d_idx.data_ptr(), self.n, self.d_type.data_ptr(),
                                          self.d_payload.data_ptr(), self.d_strbuf.data_ptr(), self.cap, C.byref(self.res), None)

    def at_pointer(self, pointers, table=True):
        return self.p.at_pointer_device(pointers, self.d_type[: self.n], self.d_payload[: self.n], self.d_strbuf, self.res.string_bytes,
                                        d_docs=self.table if table else None, ndocs=self.ndocs if table else None)


def twitter_1g():
    rows = PC.twitter_rows()
    out, size, i = [], 0, 0
    while size < (1 << 30):
        out.append(rows[i % len(rows)])
        size += len(out[-1]) + 1
        i += 1
    return b"\n".join(out) + b"\n"


def check_rows(inp, pointers, err, idx, sample=2000):
    """a seeded sample of rows against the oracle on each row's own bytes"""
    port = PO.Pointers()
    starts = inp.table[: 2 * inp.ndocs].view(-1, 2).cpu().numpy()
    err, idx = err.cpu().numpy(), idx.cpu().numpy().view(np.uint32)
    rng = random.Random(5)
    for d in rng.sample(range(inp.ndocs), min(sample, inp.ndocs)):
        b0 = int(starts[d, 1])
        b1 = int(starts[d + 1, 1]) if d + 1 < inp.ndocs else len(inp.doc)
        _r, _tw, _s, we, wi = port.table(inp.doc[b0:b1], pointers)
        for p in range(len(pointers)):
            local = int(idx[p, d]) - int(starts[d, 0]) if err[p, d] == 0 else int(idx[p, d])
            assert err[p, d] == we[p, 0] and (err[p, d] != 0 or local == wi[p, 0]), (d, pointers[p], err[p, d], we[p, 0])
    return True


def run_input(name, calls):
    if name == "twitter_1g":
        doc = twitter_1g()
        pointers = ["/id", "/user/id", "/user/screen_name", "/entities/hashtags/0/text"]
    else:
        doc = bytes(corpus.random_json(64 << 20))
        m = len(json.loads(doc))
        pointers = ["/0", f"/{m // 2}", f"/{m - 1}"]
    inp = Input(doc)
    use_table = name == "twitter_1g"
    t_s1, _ = timed(inp.stage1, calls)
    t_tab, _ = timed(inp.doc_table, calls)
    t_tok, _ = timed(inp.tokens, calls)
    t_ptr, all_ptr = timed(lambda: inp.at_pointer(pointers, use_table), calls)
    err, idx = inp.at_pointer(pointers, use_table)
    if use_table:
        ok = check_rows(inp, pointers, err, idx)
    else:
        _r, _tw, _s, we, wi = PO.Pointers().table(doc, pointers)
        ok = bool((err.cpu().numpy() == we).all() and (idx.cpu().numpy().view(np.uint32) == wi).all())
    found = int((err == 0).sum())
    inp.p.close()
    return {"input": name, "bytes": len(doc), "structurals": inp.n, "documents": inp.ndocs if use_table else 1, "pointers": len(pointers),
            "found": found, "stage1_ms": round(t_s1, 3), "doc_table_ms": round(t_tab, 3), "tokens_ms": round(t_tok, 3),
            "at_pointer_ms": round(t_ptr, 3), "at_pointer_ms_all": [round(x, 3) for x in all_ptr], "matches_oracle": ok, "calls": calls}


def sweep(lengths, calls):
    """in this process: the library SJB200_LIB names (one of the two variants); one line per length"""
    out = []
    for L in lengths:
        m = max(L // 2, 1)  # an array of m integers is about 2m structurals
        row = json.dumps(list(range(m))).encode()
        nrows = max(1, (4 << 20) // (2 * m))
        inp = Input(b"\n".join([row] * nrows) + b"\n")
        t, _ = timed(lambda: inp.at_pointer([f"/{m - 1}"]), calls)
        err, _ = inp.at_pointer([f"/{m - 1}"])
        assert int((err == 0).sum()) == inp.ndocs
        single = Input(row)
        t1, _ = timed(lambda: single.at_pointer([f"/{m - 1}"], table=False), calls)
        out.append({"structurals": inp.n // nrows, "documents": nrows, "stream_ms": round(t, 3), "one_document_ms": round(t1, 3)})
        inp.p.close()
        single.p.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--inputs", default="twitter_1g,doc_64m")
    ap.add_argument("--sweep", default="")
    ap.add_argument("--sweep-here", default="", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.sweep_here:
        print(json.dumps(sweep([int(x) for x in a.sweep_here.split(",")], a.calls)))
        return
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name in [s for s in a.inputs.split(",") if s]:
        print(json.dumps(run_input(name, a.calls)), flush=True)
    if a.sweep:
        for variant in ("warp", "cta"):
            lib = os.path.join(ROOT, "tools", "variants", f"lib_{variant}.so")
            r = subprocess.run([sys.executable, __file__, "--calls", str(a.calls), "--sweep-here", a.sweep], env=dict(os.environ, SJB200_LIB=lib),
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-2000:]
            print(json.dumps({"variant": variant, "sweep": json.loads(r.stdout.strip().splitlines()[-1])}), flush=True)


if __name__ == "__main__":
    main()
