"""Summarise one `ncu --set full` report into a small JSON file (kernel name, DRAM bytes, the kernel sources' hash).
usage: python tools/ncu_summary.py REPORT.ncu-rep OUT.json"""
import csv
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL_SOURCES = ["sjb200_scan4.cuh", "sjb200_bits.cuh", "sjb200_simt.cuh", "sjb200_params.h", "sjb200_kernels.cu", "sjb200_utf8.cuh"]  # same list as bench.py


def kernel_source_hash():
    h = hashlib.sha256()
    for f in KERNEL_SOURCES:
        with open(os.path.join(ROOT, "simdjson_b200", "csrc", f), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()[:16]

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_bytes.sum", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__cycles_active.avg",
    "sm__cycles_elapsed.max",
]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    res = []
    for vals in rows[2:]:
        d = {"Kernel Name": vals[hdr.index("Kernel Name")], "kernel_src_sha16": kernel_source_hash()}
        for i, h in enumerate(hdr):
            if h in KEYS or ("issue_stalled" in h and h.endswith("per_issue_active.ratio")):
                d[h] = [vals[i], units[i]]
        res.append(d)
    json.dump(res if len(res) > 1 else res[0], open(out, "w"), indent=1)
    print("wrote", out, "kernels:", [r["Kernel Name"][:60] for r in res])


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
