"""The stage-2 grammar on the device (sjb200_document_errors_dev), timed next to sjb200_tokens_dev on the same input.
Inputs:
  twitter_1g  1 GiB of NDJSON rows, the statuses of twitter.json repeated, with the device document table
  doc_64m     the 64 MiB corpus.random_json document
  deep_64m    ~64 MiB array of documents nested 1 000 deep (max_depth 1024)
Every time is the median over --calls calls after one warm-up, CUDA events around the call (each call ends in its own
synchronise).  Every input is valid JSON, so every verdict must be SUCCESS, and the SUCCESS index of each document is
checked against the document table.  Prints the GPU's name, power limit and SM clock, then one JSON line per input.

    python tools/document_errors_bench.py [--calls 10] [--inputs twitter_1g,doc_64m,deep_64m]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import pointer_cases as PC  # noqa: E402
from pointer_bench import gpu_info, timed  # noqa: E402
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import capi, corpus  # noqa: E402


def make(name):
    if name == "twitter_1g":
        base = PC.stream_of(PC.twitter_rows())
        return (base * ((1 << 30) // len(base) + 1))[: 1 << 30].rsplit(b"\n", 1)[0] + b"\n", True
    if name == "doc_64m":
        return bytes(corpus.random_json(64 << 20, seed=5)), False
    if name == "deep_64m":
        one = b"[" * 1000 + b'{"a":[1,2,{}],"b":"x"}' + b"]" * 1000
        return b"[" + b",".join([one] * ((64 << 20) // (len(one) + 1))) + b"]", False
    raise ValueError(name)


def bench(name, calls):
    doc, stream = make(name)
    d = torch.from_numpy(np.frombuffer(doc, dtype=np.uint8).copy()).cuda()
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(len(doc), 1024)
    assert rc == sj.SUCCESS
    assert p.stage1_device(d, sj.REGULAR) == sj.SUCCESS
    n = p.n_structural_indexes
    d_idx = p.device_index_buffer()
    cap = int(sj.lib().sjb200_string_buf_capacity(len(doc)))
    d_type = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_payload = torch.empty(n, dtype=torch.int64, device="cuda")
    d_strbuf = torch.empty(cap, dtype=torch.uint8, device="cuda")
    tres = capi.TokensResult()
    L = sj.lib()

    def tokens():
        return L.sjb200_tokens_dev(p._ctx, d.data_ptr(), len(doc), d_idx.data_ptr(), n, d_type.data_ptr(), d_payload.data_ptr(), d_strbuf.data_ptr(), cap,
                                   C.byref(tres), None)

    assert tokens() == 0
    table, nd = None, 1
    if stream:
        table = torch.empty(2 * (n + 1), dtype=torch.int32, device="cuda")
        ndc = C.c_uint32(0)
        assert L.sjb200_document_table_dev(p._ctx, d.data_ptr(), d_idx.data_ptr(), n, table.data_ptr(), n + 1, C.byref(ndc), None) == 0
        nd = ndc.value
    out = torch.empty((nd, 2), dtype=torch.int32, device="cuda")
    res = capi.DocumentErrorsResult()

    def verdicts():
        return L.sjb200_document_errors_dev(p._ctx, d_type.data_ptr(), d_payload.data_ptr(), n, None if table is None else table.data_ptr(),
                                            nd if stream else 0, 1024, out.data_ptr(), C.byref(res), None)

    assert verdicts() == 0
    o = out.cpu().numpy()
    assert res.ndocs_in_error == 0 and (o[:, 0] == 0).all(), (res.ndocs_in_error, res.first_doc_in_error)
    ends = np.append(table[2: 2 * nd: 2].cpu().numpy(), n) if stream else np.array([n])
    assert np.array_equal(o[:, 1].view(np.uint32), ends.astype(np.uint32))
    t_tok = timed(tokens, calls)[0]
    t_err = timed(verdicts, calls)[0]
    p.close()
    return {"input": name, "bytes": len(doc), "structurals": n, "documents": nd, "document_errors_ms": round(t_err, 3), "tokens_ms": round(t_tok, 3),
            "ratio": round(t_err / t_tok, 3), "structurals_per_ns": round(n / (t_err * 1e6), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--inputs", default="twitter_1g,doc_64m,deep_64m")
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}))
    for name in a.inputs.split(","):
        print(json.dumps(bench(name, a.calls)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
