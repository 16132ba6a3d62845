"""Float columns on the device (sjb200_column_double_dev), timed on one GPU:
  floats_1g  1 GiB of seeded NDJSON rows {"price": shortest double, "rating": one decimal, "id": int, "name": string}
             (a pool of 65 536 rows repeated): get_double of /price and /rating against sjb200_column_dev INT64 of /id,
             the same rows
  slow_256m  256 MiB of rows {"v": a number of 20-25 significant digits}: every value needs more than its first 19
             digits (Eisel-Lemire on w and w + 1, the exact comparison when they disagree)
  big_16m    four rows, one holding a 16 MiB number (summarized by one CTA)
Every time is the median over --calls raw calls into preallocated outputs after a warm-up, CUDA events around the call
(each call ends in its own synchronise).  Values are checked bit for bit against float() of each sampled row's text.
Prints the GPU's name, power limit and SM clock, then one JSON line per input.
    python tools/column_double_bench.py [--calls 10] [--inputs floats_1g,slow_256m,big_16m]
"""
import argparse
import ctypes as C
import json
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import double_cases as DC  # noqa: E402
import pointer_bench as PB  # noqa: E402
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import capi  # noqa: E402


def repeat_to(rows, size):
    block = b"\n".join(rows) + b"\n"
    k = max(1, size // len(block))
    return block * k, len(rows) * k


def floats_pool(seed=1):
    rng = np.random.default_rng(seed)
    prices = rng.lognormal(3, 1.5, 65536) * np.where(rng.random(65536) < 0.5, 1.0, 1e-3)
    ratings = np.round(rng.uniform(1, 5, 65536), 1)
    texts = [(repr(float(p)), repr(float(r))) for p, r in zip(prices, ratings)]
    rows = [f'{{"price":{p},"rating":{r},"id":{i * 7919 + 13},"name":"item {i}"}}'.encode() for i, (p, r) in enumerate(texts)]
    return rows, texts


def slow_pool(seed=2):
    texts = DC.slow_heavy(65536, seed)
    return [f'{{"v":{t}}}'.encode() for t in texts], [(t,) for t in texts]


class DoubleColumn:
    def __init__(self, inp, rows):
        self.inp, self.rows, self.R = inp, rows, rows.shape[0]
        self.err = torch.empty(self.R, dtype=torch.int32, device="cuda")
        self.rt = torch.empty(self.R, dtype=torch.uint8, device="cuda")
        self.vals = torch.empty(self.R, dtype=torch.float64, device="cuda")
        self.out = capi.ColumnResult()

    def call(self):
        i = self.inp
        return sj.lib().sjb200_column_double_dev(i.p._ctx, i.d.data_ptr(), i.d.numel(), i.d_idx.data_ptr(), i.d_type.data_ptr(), i.d_payload.data_ptr(), i.n,
                                                 self.rows.data_ptr(), self.R, self.err.data_ptr(), self.rt.data_ptr(), self.vals.data_ptr(),
                                                 C.byref(self.out), None)


class IntColumn:
    def __init__(self, inp, rows):
        self.inp, self.rows, self.R = inp, rows, rows.shape[0]
        self.err = torch.empty(self.R, dtype=torch.int32, device="cuda")
        self.rt = torch.empty(self.R, dtype=torch.uint8, device="cuda")
        self.vals = torch.empty(self.R, dtype=torch.int64, device="cuda")
        self.out = capi.ColumnResult()

    def call(self):
        i = self.inp
        return sj.lib().sjb200_column_dev(i.p._ctx, capi.COLUMN_INT64, i.d_type.data_ptr(), i.d_payload.data_ptr(), i.n, i.d_strbuf.data_ptr(),
                                          i.res.string_bytes, self.rows.data_ptr(), self.R, self.err.data_ptr(), self.rt.data_ptr(), self.vals.data_ptr(),
                                          None, None, 0, C.byref(self.out), None)


def matches(col, texts, field, sample=1500):
    """a seeded sample of rows (row d is texts[d % len(texts)]) against float() of its text"""
    err = col.err.cpu().numpy()
    bits = col.vals.view(torch.int64).cpu().numpy().view(np.uint64)
    rng = random.Random(7)
    for d in rng.sample(range(col.R), min(sample, col.R)):
        if (int(err[d]), int(bits[d])) != DC.expect(texts[d % len(texts)][field]):
            return False
    return True


def run_rows(name, rows, texts, size, fields, calls, int_pointer=None):
    doc, nrows = repeat_to(rows, size)
    inp = PB.Input(doc)
    pointers = [p for p, _f in fields] + ([int_pointer] if int_pointer else [])
    perr, pidx = inp.at_pointer(pointers)
    out = []
    for k, (pointer, field) in enumerate(fields):
        col = DoubleColumn(inp, torch.stack((perr[k], pidx[k]), -1).contiguous())
        assert col.call() == 0
        t, all_ms = PB.timed(col.call, calls)
        out.append({"pointer": pointer, "kind": "get_double", "rows": col.R, "rows_in_error": col.out.rows_in_error, "call_ms": round(t, 3),
                    "call_ms_all": [round(x, 3) for x in all_ms], "matches_float": matches(col, texts, field)})
    if int_pointer:
        col = IntColumn(inp, torch.stack((perr[-1], pidx[-1]), -1).contiguous())
        assert col.call() == 0
        t, all_ms = PB.timed(col.call, calls)
        out.append({"pointer": int_pointer, "kind": "INT64", "rows": col.R, "rows_in_error": col.out.rows_in_error, "call_ms": round(t, 3),
                    "call_ms_all": [round(x, 3) for x in all_ms]})
    res = {"input": name, "bytes": len(doc), "structurals": inp.n, "documents": inp.ndocs, "columns": out, "calls": calls}
    inp.p.close()
    return res


def run_floats(calls):
    rows, texts = floats_pool()
    return run_rows("floats_1g", rows, texts, 1 << 30, [("/price", 0), ("/rating", 1)], calls, int_pointer="/id")


def run_slow(calls):
    rows, texts = slow_pool()
    return run_rows("slow_256m", rows, texts, 256 << 20, [("/v", 0)], calls)


def run_big(calls):
    h = DC.halfway(1.0)
    big = h + "0" * ((16 << 20) - len(h)) + "1"
    texts = [("1.5",), (big,), ("-0.0",), ("2.5e-3",)]
    rows = [f'{{"v":{t[0]}}}'.encode() for t in texts]
    inp = PB.Input(b"\n".join(rows) + b"\n")
    perr, pidx = inp.at_pointer(["/v"])
    col = DoubleColumn(inp, torch.stack((perr[0], pidx[0]), -1).contiguous())
    assert col.call() == 0
    t, all_ms = PB.timed(col.call, calls)
    bits = col.vals.view(torch.int64).cpu().numpy().view(np.uint64).tolist()
    ok = bits == [DC.bits(1.5), DC.bits(1.0) + 1, DC.bits(-0.0), DC.bits(2.5e-3)]
    res = {"input": "big_16m", "bytes": inp.d.numel(), "rows": col.R, "call_ms": round(t, 3), "call_ms_all": [round(x, 3) for x in all_ms],
           "matches_float": ok, "calls": calls}
    inp.p.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--inputs", default="floats_1g,slow_256m,big_16m")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "column_double_bench needs a GPU"
    print(json.dumps({"gpu": PB.gpu_info()}), flush=True)
    for name in a.inputs.split(","):
        run = {"floats_1g": run_floats, "slow_256m": run_slow, "big_16m": run_big}[name]
        print(json.dumps(run(a.calls)), flush=True)


if __name__ == "__main__":
    main()
