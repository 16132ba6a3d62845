"""Tuning probe: stage-1 kernel time of ONE build variant (SJB200_LIB) on the bench document, with whole-buffer parity.
The document and the oracle's answer are cached in /tmp so that a series of variants pays for them once.
  PROBE_BYTES (default 64 MiB), PROBE_TAG, PROBE_PARITY=0 skips the comparison (ablation builds)."""
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

size = int(os.environ.get("PROBE_BYTES", 64 << 20))
tag = os.environ.get("PROBE_TAG") or os.path.basename(os.environ.get("SJB200_LIB", "default"))
cache = f"/tmp/probe_cache_{size}.npz"
noparity = os.environ.get("PROBE_PARITY", "1") == "0"
if noparity and not os.path.exists(cache):
    doc, words, want_err, want_n = corpus.random_json(size).copy(), None, 0, None
elif os.path.exists(cache):
    z = np.load(cache)
    doc, words, want_err, want_n = z["doc"], z["words"], int(z["err"]), int(z["n"])
else:
    import oracle_lib as O
    doc = corpus.random_json(size).copy()
    w = O.Port().stage1(doc, 0)
    words, want_err, want_n = w.words().copy(), int(w.err), int(w.n)
    np.savez(cache, doc=doc, words=words, err=want_err, n=want_n)
rc, p = sj.get_active_implementation().create_dom_parser_implementation(len(doc))
assert rc == 0, rc
p.set_option("time_kernel", 1)
d = torch.from_numpy(doc).cuda()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
if os.environ.get("PROBE_FORCE_GRID"):
    p.set_option("force_grid", int(os.environ["PROBE_FORCE_GRID"]))
rc = p.stage1_device(d, 0)
if want_n is None:
    want_n = p.n_structural_indexes
res = {"tag": tag, "bytes": size}
if not noparity:
    got = p.device_index_buffer().cpu().numpy().view(np.uint32)
    res["parity"] = bool(rc == want_err and p.n_structural_indexes == want_n and np.array_equal(got[: want_n + 3], words))
warm, cold = [], []
for it in range(8):
    p.stage1_device(d, 0)
    warm.append(p.get_stat("kernel_ms"))
for it in range(6):
    flush.fill_(it)  # 256 MiB > L2: the next launch finds nothing of its input or of the descriptors in L2
    torch.cuda.synchronize()
    p.stage1_device(d, 0)
    cold.append(p.get_stat("kernel_ms"))
alg = size + 4 * want_n + 12
res.update({"warm_ms": min(warm[2:]), "cold_ms": min(cold[1:]), "cold_med_ms": sorted(cold[1:])[len(cold[1:]) // 2],
            "in_gbs_cold": size / min(cold[1:]) / 1e6, "alg_frac_cold": alg / min(cold[1:]) / 1e6 / PEAK_GBS})
print(json.dumps(res), flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
with open(os.path.join(ROOT, "gpurun_out", "probe2.jsonl"), "a") as f:
    f.write(json.dumps(res) + "\n")
