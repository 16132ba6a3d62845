"""Time sharded stage 1 of an NDJSON stream: stage1_sharded_stream(STREAMING_FINAL) against plain stage1_sharded on the
same shards, alternated pass by pass in one session, and sjb200_document_table_shard_dev on the result.

  python tools/sharded_stream_bench.py [--mib 1024] [--ranks 4] [--steps 20]

All ranks run as threads of this process on one GPU (connect_local), so the ranks' scans share that GPU's SMs and HBM: a
pass here costs about what one pass over the whole buffer costs, plus the exchange rounds.  A pass's time is the slowest
rank's host wall-clock from enqueue to the return of finish.  Prints the card's name and power limit with the numbers."""
import argparse
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import corpus, sharding  # noqa: E402


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--ranks", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    doc = corpus.ndjson_rows(a.mib << 20)
    cuts = sharding.shard_cuts_at_lines(doc, a.ranks)
    world = a.ranks
    impl = sj.get_active_implementation(0)
    parsers, comms, shards, idx = [], [], [], []
    L = sj.lib()
    for r in range(world):
        n = cuts[r + 1] - cuts[r]
        rc, p = impl.create_dom_parser_implementation(n)
        assert rc == sj.SUCCESS
        parsers.append(p)
        comms.append(sharding.Comm(p, r, world))
        shards.append(torch.from_numpy(doc[cuts[r]: cuts[r + 1]].copy()).cuda())
        idx.append(torch.empty(int(L.sjb200_index_words(n)), dtype=torch.int32, device="cuda"))
    sharding.Comm.connect_local(comms)
    streams = [torch.cuda.Stream() for _ in range(world)]
    results = [None] * world
    barrier = threading.Barrier(world)

    def one_pass(r, kind):
        barrier.wait()
        t0 = time.perf_counter()
        if kind == "stream":
            rc, x = comms[r].scan_stream(shards[r], idx[r], r == world - 1, sj.STREAMING_FINAL, streams[r])
        else:
            rc, x = comms[r].scan(shards[r], idx[r], r == world - 1, streams[r])
        streams[r].synchronize()
        results[r] = (rc, time.perf_counter() - t0, x)

    def run(kind):
        th = [threading.Thread(target=one_pass, args=(r, kind)) for r in range(world)]
        [t.start() for t in th]
        [t.join() for t in th]
        assert all(res[0] == 0 for res in results), [res[0] for res in results]
        return max(res[1] for res in results)

    times = {"plain": [], "stream": []}
    for step in range(a.warmup + a.steps):
        for kind in ("plain", "stream"):  # alternated: both see the same clocks and temperature
            t = run(kind)
            if step >= a.warmup:
                times[kind].append(t)
    res = [results[r][2] for r in range(world)]  # the last stream pass
    # document tables: CUDA events around each rank's call, ranks one after the other
    tab_ms = []
    for r in range(world):
        for k in range(a.warmup + a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(streams[r])
            comms[r].document_table(shards[r], idx[r], res[r], streams[r])
            e1.record(streams[r])
            e1.synchronize()
            if k >= a.warmup:
                tab_ms.append((r, e0.elapsed_time(e1)))
    gb = len(doc) / 1e9
    med = {k: statistics.median(v) for k, v in times.items()}
    print(f"device: {power_limit()}")
    print(f"input: {len(doc)} bytes NDJSON, {world} ranks as threads on one GPU, {a.steps} passes of each kind, alternated")
    for k in ("plain", "stream"):
        print(f"  stage1_sharded{'_stream(STREAMING_FINAL)' if k == 'stream' else ''}: median {med[k] * 1e3:.3f} ms  "
              f"(min {min(times[k]) * 1e3:.3f}, max {max(times[k]) * 1e3:.3f})  {gb / med[k]:.1f} GB/s")
    print(f"  extra cost of the stream finish: {(med['stream'] - med['plain']) * 1e3:.3f} ms per pass (median difference)")
    per_rank = {r: statistics.median([t for q, t in tab_ms if q == r]) for r in range(world)}
    print("  document_table_shard_dev per rank, median ms: " + ", ".join(f"r{r} {per_rank[r]:.3f} ({int(res[r].kept)} structurals)" for r in range(world)))
    for c in comms:
        c.close()
    for p in parsers:
        p.close()


if __name__ == "__main__":
    main()
