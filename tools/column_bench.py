"""Typed columns on the device (sjb200_column_dev), timed on the inputs of tools/pointer_bench.py:
  twitter_1g  1 GiB of NDJSON rows, the statuses of twitter.json repeated: every kind on its row pointers
  doc_64m     the 64 MiB corpus.random_json document: ARRAY_SIZE of "" against sjb200_at_pointer_dev of its last root
              element (both walk the same structurals, one CTA each; both raw calls into preallocated outputs)
  long_512m   512 MiB of NDJSON rows {"b": string} with strings of 4-40 KiB (and one row in 8 with a short one): the
              STRING column of /b, whose long strings are copied chunk by chunk by the long-string kernel
Every time is the median over --calls calls after a warm-up, CUDA events around the call (each call ends in its own
synchronise).  For the STRING columns also the kernels' time from torch.profiler (a separate run) and the bytes the
column needs to read and write over it -- memory bound, against the H100 SXM data sheet's 3.35 TB/s of HBM3.  Outputs are
checked against the oracle (sjo_column) on a seeded sample of rows, the whole document.  Prints the GPU's name, power limit
and SM clock, then one JSON line per input.
    python tools/column_bench.py [--calls 10] [--inputs twitter_1g,doc_64m]
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

import column_oracle as CO  # noqa: E402
import pointer_bench as PB  # noqa: E402
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import capi, corpus  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet
KIND_NAMES = {capi.COLUMN_INT64: "INT64", capi.COLUMN_UINT64: "UINT64", capi.COLUMN_BOOL: "BOOL", capi.COLUMN_STRING: "STRING",
              capi.COLUMN_ARRAY_SIZE: "ARRAY_SIZE", capi.COLUMN_OBJECT_SIZE: "OBJECT_SIZE"}
TWITTER = [("/id", capi.COLUMN_INT64), ("/id", capi.COLUMN_UINT64), ("/user/id", capi.COLUMN_INT64), ("/user/id", capi.COLUMN_UINT64),
           ("/user/screen_name", capi.COLUMN_STRING), ("/text", capi.COLUMN_STRING), ("/favorited", capi.COLUMN_BOOL),
           ("/entities/hashtags", capi.COLUMN_ARRAY_SIZE), ("/user", capi.COLUMN_OBJECT_SIZE), ("/retweeted_status/id", capi.COLUMN_INT64)]


class Column:
    """one pointer's rows of an Input and preallocated outputs: call() is one sjb200_column_dev"""

    def __init__(self, inp, rows, kind, string_bytes=0):
        self.inp, self.rows, self.kind = inp, rows, kind
        R = rows.shape[0]
        self.R = R
        self.err = torch.empty(R, dtype=torch.int32, device="cuda")
        self.rt = torch.empty(R, dtype=torch.uint8, device="cuda")
        self.vals = torch.empty(R, dtype=torch.int64, device="cuda")
        self.offs = torch.empty(R + 1, dtype=torch.int64, device="cuda")
        self.bytes = torch.empty(max(string_bytes, 1), dtype=torch.uint8, device="cuda")
        self.cap = string_bytes
        self.out = capi.ColumnResult()

    def call(self):
        i, st = self.inp, self.kind == capi.COLUMN_STRING
        return sj.lib().sjb200_column_dev(i.p._ctx, self.kind, i.d_type.data_ptr(), i.d_payload.data_ptr(), i.n, i.d_strbuf.data_ptr(), i.res.string_bytes,
                                          self.rows.data_ptr(), self.R, self.err.data_ptr(), self.rt.data_ptr(), None if st else self.vals.data_ptr(),
                                          self.offs.data_ptr() if st else None, self.bytes.data_ptr() if st else None, self.cap, C.byref(self.out), None)


def kernel_ms(fn, calls):
    """mean device time per call of the column kernels (and the tile scan), from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "col_" in e.key or "tile_scan" in e.key)
    return us / 1000.0 / calls


def check_sample(inp, pointer, kind, col, sample=1500):
    """a seeded sample of rows against the oracle on each row's own bytes"""
    cols = CO.Columns()
    starts = inp.table[: 2 * inp.ndocs].view(-1, 2).cpu().numpy()
    err, rt = col.err.cpu().numpy(), col.rt.cpu().numpy()
    vals = col.vals.cpu().numpy().view(np.uint64)
    offs = col.offs.cpu().numpy()
    data = bytes(col.bytes[: col.out.string_bytes].cpu().numpy()) if kind == capi.COLUMN_STRING else b""
    rng = random.Random(7)
    for d in rng.sample(range(inp.ndocs), min(sample, inp.ndocs)):
        b0 = int(starts[d, 1])
        b1 = int(starts[d + 1, 1]) if d + 1 < inp.ndocs else len(inp.doc)
        _tab, we, wt, wv, ws = cols.of_document(kind, inp.doc[b0:b1], [pointer])
        if err[d] != we[0, 0] or rt[d] != wt[0, 0]:
            return False
        if kind == capi.COLUMN_STRING:
            if data[offs[d]: offs[d + 1]] != ws[0]:
                return False
        elif int(vals[d] if kind != capi.COLUMN_BOOL else col.vals.view(torch.uint8)[d].item()) != int(wv[0, 0]):
            return False
    return True


def string_column(inp, pointer, calls):
    """the STRING column of one pointer over the rows of inp: call and kernel times, bytes moved"""
    perr, pidx = inp.at_pointer([pointer])
    rows = torch.stack((perr[0], pidx[0]), -1).contiguous()
    col = Column(inp, rows, capi.COLUMN_STRING)
    assert col.call() in (0, capi.CAPACITY)
    need = col.out.string_bytes
    col = Column(inp, rows, capi.COLUMN_STRING, need)
    assert col.call() == 0
    t, all_ms = PB.timed(col.call, calls)
    k = kernel_ms(col.call, calls)
    moved = 34 * col.R + 8 + 2 * need  # rows 8, type 1, payload 8, length word 4, err 4, row type 1, offset 8 per row; the bytes in and out
    r = {"pointer": pointer, "kind": "STRING", "rows": col.R, "rows_in_error": col.out.rows_in_error, "call_ms": round(t, 3),
         "call_ms_all": [round(x, 3) for x in all_ms], "matches_oracle": check_sample(inp, pointer, capi.COLUMN_STRING, col),
         "string_bytes": need, "kernel_ms": round(k, 3), "bytes_moved": moved, "kernel_TBps": round(moved / (k * 1e-3) / 1e12, 3),
         "bound": "memory (HBM3)", "share_of_3.35TBps": round(moved / (k * 1e-3) / 1e12 / HBM_TBS, 3)}
    return r


def long_512m():
    rng = np.random.default_rng(3)
    pool = "".join(chr(c) for c in rng.integers(0x20, 0x7F, 64 << 10)).replace("\\", "/").replace('"', "'")
    out, size, i = [], 0, 0
    while size < (512 << 20):
        n = int(rng.integers(4096, 40960)) if i % 8 else 12
        o = int(rng.integers(0, len(pool) - n))
        out.append(json.dumps({"b": pool[o: o + n], "i": i}).encode())
        size += len(out[-1]) + 1
        i += 1
    return b"\n".join(out) + b"\n"


def run_long(calls):
    inp = PB.Input(long_512m())
    r = string_column(inp, "/b", calls)
    res = {"input": "long_512m", "bytes": len(inp.doc), "structurals": inp.n, "documents": inp.ndocs, "columns": [r], "calls": calls}
    inp.p.close()
    return res


def run_twitter(calls):
    inp = PB.Input(PB.twitter_1g())
    pointers = sorted({p for p, _k in TWITTER})
    perr, pidx = inp.at_pointer(pointers)
    out = []
    for pointer, kind in TWITTER:
        if kind == capi.COLUMN_STRING:
            out.append(string_column(inp, pointer, calls))
            continue
        p = pointers.index(pointer)
        rows = torch.stack((perr[p], pidx[p]), -1).contiguous()
        col = Column(inp, rows, kind)
        assert col.call() == 0
        t, all_ms = PB.timed(col.call, calls)
        out.append({"pointer": pointer, "kind": KIND_NAMES[kind], "rows": col.R, "rows_in_error": col.out.rows_in_error, "call_ms": round(t, 3),
                    "call_ms_all": [round(x, 3) for x in all_ms], "matches_oracle": check_sample(inp, pointer, kind, col)})
    res = {"input": "twitter_1g", "bytes": len(inp.doc), "structurals": inp.n, "documents": inp.ndocs, "columns": out, "calls": calls}
    inp.p.close()
    return res


def run_doc(calls):
    doc = bytes(corpus.random_json(64 << 20))
    m = len(json.loads(doc))
    inp = PB.Input(doc)
    perr, pidx = inp.at_pointer([""], table=False)
    rows = torch.stack((perr[0], pidx[0]), -1).contiguous()
    col = Column(inp, rows, capi.COLUMN_ARRAY_SIZE)
    assert col.call() == 0
    t_size, all_size = PB.timed(col.call, calls)
    # sjb200_at_pointer_dev of the last element, a raw call into a preallocated output like the column's
    last = f"/{m - 1}".encode()
    buf = C.create_string_buffer(last, len(last))
    ptrs = (C.c_void_p * 1)(C.addressof(buf))
    lens = (C.c_size_t * 1)(len(last))
    pout = torch.empty(2, dtype=torch.int32, device="cuda")

    def at_pointer():
        return sj.lib().sjb200_at_pointer_dev(inp.p._ctx, inp.d_type.data_ptr(), inp.d_payload.data_ptr(), inp.n, inp.d_strbuf.data_ptr(),
                                              inp.res.string_bytes, None, 0, ptrs, lens, 1, pout.data_ptr(), None)
    assert at_pointer() == 0
    t_ptr, all_ptr = PB.timed(at_pointer, calls)
    ok = int(col.err[0]) == 0 and int(col.vals[0]) == min(m, 0xFFFFFF) and int(pout[0]) == 0
    res = {"input": "doc_64m", "bytes": len(doc), "structurals": inp.n, "root_elements": m, "array_size_ms": round(t_size, 3),
           "array_size_ms_all": [round(x, 3) for x in all_size], "at_pointer_last_ms": round(t_ptr, 3),
           "at_pointer_last_ms_all": [round(x, 3) for x in all_ptr], "matches_oracle": ok, "calls": calls}
    inp.p.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--inputs", default="twitter_1g,doc_64m,long_512m")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "column_bench needs a GPU"
    print(json.dumps({"gpu": PB.gpu_info()}), flush=True)
    for name in a.inputs.split(","):
        run = {"twitter_1g": run_twitter, "doc_64m": run_doc, "long_512m": run_long}[name]
        print(json.dumps(run(a.calls)), flush=True)


if __name__ == "__main__":
    main()
