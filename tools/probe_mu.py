"""Tuning probe: minify (both kernels) and validate_utf8 kernel times at PROBE_BYTES (default 256 MiB), whole-buffer parity.
Inputs and the oracle's answers are cached in /tmp."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import corpus  # noqa: E402
from bench import peaks  # noqa: E402

PEAK_GBS = peaks()[0]  # MEASURED_PEAKS.json hbm_gbs, else the data sheet's figure

size = int(os.environ.get("PROBE_BYTES", 256 << 20))
tag = os.environ.get("PROBE_TAG") or os.path.basename(os.environ.get("SJB200_LIB", "default"))
cache = f"/tmp/probe_mu_cache_{size}.npz"
if os.path.exists(cache):
    z = np.load(cache)
    j, wout, werr, u = z["j"], z["wout"], int(z["werr"]), z["u"]
else:
    import oracle_lib as O
    j = corpus.random_json(size, pretty_bias=0.8, utf8_rate=0.15).copy()
    werr, wo = O.Port().minify(j)
    wout = np.frombuffer(wo, dtype=np.uint8).copy()
    u = corpus.random_utf8(size).copy()
    np.savez(cache, j=j, wout=wout, werr=werr, u=u)
rc, p = sj.get_active_implementation().create_dom_parser_implementation(len(j))
assert rc == 0
p.set_option("time_kernel", 1)
dj = torch.from_numpy(j).cuda()
dst = torch.empty(len(j), dtype=torch.uint8, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
res = {"tag": tag, "bytes": size}
for mk in (4,):
    dst.zero_()
    rcm, dl = p.minify_device(dj, dst)
    same = bool(rcm == werr and dl == len(wout) and torch.equal(dst[:dl].cpu(), torch.from_numpy(wout)))
    ts = []
    for it in range(5):
        flush.fill_(it)
        torch.cuda.synchronize()
        p.minify_device(dj, dst)
        ts.append(p.get_stat("kernel_ms"))
    t = min(ts[1:])
    res[f"minify_k{mk}"] = {"parity": same, "ms": t, "in_gbs": size / t / 1e6, "kept": dl / size, "alg_frac": (size + dl) / t / 1e6 / PEAK_GBS}
du = torch.from_numpy(u).cuda()
ts = []
for it in range(5):
    flush.fill_(it)
    torch.cuda.synchronize()
    r = p.validate_utf8_device(du)
    ts.append(p.get_stat("kernel_ms"))
t = min(ts[1:])
res["utf8"] = {"valid": int(r), "ms": t, "in_gbs": size / t / 1e6, "frac": size / t / 1e6 / PEAK_GBS}
ts = []
for it in range(5):
    flush.fill_(it)
    torch.cuda.synchronize()
    r2 = p.validate_utf8_device(dj)
    ts.append(p.get_stat("kernel_ms"))
t = min(ts[1:])
res["utf8_on_json"] = {"valid": int(r2), "ms": t, "in_gbs": size / t / 1e6, "frac": size / t / 1e6 / PEAK_GBS}
print(json.dumps(res), flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
with open(os.path.join(ROOT, "gpurun_out", "probe_mu.jsonl"), "a") as f:
    f.write(json.dumps(res) + "\n")
