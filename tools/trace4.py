"""Where a scan warp's time goes (trace build of scan4, -DSJB200_SCAN4_TRACE=1: SM cycle counter at the phase
boundaries of scan warps 0 and 9, kept in shared memory and dumped at kernel exit -- no global stores in the loop).
  SJB200_LIB=tools/variants/lib_trace.so python tools/trace4.py"""
import os
import sys

import numpy as np
import pynvml
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import corpus  # noqa: E402

size = int(os.environ.get("PROBE_BYTES", 64 << 20))
doc = corpus.random_json(size).copy()
rc, p = sj.get_active_implementation().create_dom_parser_implementation(len(doc))
p.set_option("debug_timeline", 1)
p.set_option("time_kernel", 1)
d = torch.from_numpy(doc).cuda()
for _ in range(3):
    p.stage1_device(d, 0)
kms = p.get_stat("kernel_ms")
rows = 4096
buf = np.zeros((rows, 8), dtype=np.uint64)
n = sj.lib().sjb200_get_debug_timeline(p._ctx, buf.ctypes.data, rows)
IT, PTS = 8, 12
names = ["top", "ticket", "load issued", "data here", "boundary", "scanned", "arrive/compose", "publish", "resolved seen", "emitted"]
ctas = []
for c in range(torch.cuda.get_device_properties(0).multi_processor_count):  # one CTA per SM
    r = buf[c * (1 + 2 * IT): (c + 1) * (1 + 2 * IT)]
    if r[0, 0] == 0:
        continue
    tr = np.zeros((2, IT, PTS), dtype=np.int64)
    for a in range(2):
        for b in range(IT):
            q = r[1 + a * IT + b]
            for k in range(6):
                tr[a, b, 2 * k] = int(q[k]) & 0xFFFFFFFF
                tr[a, b, 2 * k + 1] = int(q[k]) >> 32
    ctas.append((c, [int(x) for x in r[0, :5]], tr))
t_entry = np.array([c[1][0] for c in ctas], dtype=np.int64)
t_roles = np.array([c[1][1] for c in ctas], dtype=np.int64)
t_done = np.array([c[1][2] for c in ctas], dtype=np.int64)
t_exit = np.array([c[1][3] for c in ctas], dtype=np.int64)
t0 = t_entry.min()
print(f"kernel_ms (events) {kms:.4f}; CTAs {len(ctas)}")
print(f"CTA entry: first 0.00, last {(t_entry.max()-t0)/1e3:.2f} us; roles start mean {(t_roles-t0).mean()/1e3:.2f}; scan role done mean {(t_done-t0).mean()/1e3:.2f} max {(t_done.max()-t0)/1e3:.2f}; exit max {(t_exit.max()-t0)/1e3:.2f} us")
pynvml.nvmlInit()
clk = float(pynvml.nvmlDeviceGetMaxClockInfo(pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device()), pynvml.NVML_CLOCK_SM))  # cycles per us
for a, wname in ((0, "warp 0"), (1, "warp 9")):
    print(f"-- {wname}: mean cycles between consecutive points, per iteration (us at the maximum SM clock, {clk:.0f} MHz, in brackets)")
    for b in range(IT):
        segs = []
        for k in range(1, 10):
            v = [((c[2][a, b, k] - c[2][a, b, k - 1]) & 0xFFFFFFFF) for c in ctas if c[2][a, b, k] and c[2][a, b, k - 1]]
            segs.append(np.mean(v) if v else float("nan"))
        tot = [((c[2][a, b + 1, 0] - c[2][a, b, 0]) & 0xFFFFFFFF) for c in ctas if b + 1 < IT and c[2][a, b + 1, 0] and c[2][a, b, 0]]
        print(f"it{b}: " + " ".join(f"{names[k]}={s:.0f}" for k, s in zip(range(1, 10), segs)) + (f" | iteration {np.mean(tot):.0f} cyc [{np.mean(tot)/clk:.2f} us]" if tot else ""))
