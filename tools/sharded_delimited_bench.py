"""Time sharded stage 1 of RS-delimited and comma-delimited streams: sjb200_stage1_sharded_delimited in modes 3-6 on
NDJSON rows written as an RS stream (RS row LF) and comma-joined (row ,LF), against the mode-2 stream pass on the same
rows as NDJSON and the single-GPU sjb200_stage1_dev in modes 4 and 6, alternated pass by pass in one session.

  python tools/sharded_delimited_bench.py [--mib 1024] [--ranks 4] [--steps 10]

All ranks run as threads of this process on one GPU (connect_local) and the cuts lie right after line feeds.  A sharded
pass's time is the slowest rank's host wall-clock from enqueue to the return of finish; a single-GPU pass's is the host
wall-clock of sjb200_stage1_dev.  Prints the card's name, power limit and SM clock with the medians."""
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


def device_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--ranks", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    rows = [r for r in bytes(corpus.ndjson_rows(a.mib << 20)).split(b"\n") if r]
    docs = {"ndjson": b"\n".join(rows) + b"\n", "rs": b"".join(b"\x1e" + r + b"\n" for r in rows), "comma": b",\n".join(rows)}
    world = a.ranks
    impl = sj.get_active_implementation(0)
    L = sj.lib()
    cap = max(len(d) for d in docs.values())
    shards, cuts_of = {}, {}
    for name, doc in docs.items():
        arr = np.frombuffer(doc, dtype=np.uint8)
        cuts = sharding.shard_cuts_at_lines(arr, world)
        cuts_of[name] = cuts
        shards[name] = [torch.from_numpy(arr[cuts[r]: cuts[r + 1]].copy()).cuda() for r in range(world)]
    parsers, comms, idx = [], [], []
    for r in range(world):
        n = max(int(s[r].numel()) for s in shards.values())
        rc, p = impl.create_dom_parser_implementation(n)
        assert rc == sj.SUCCESS
        parsers.append(p)
        comms.append(sharding.Comm(p, r, world))
        idx.append(torch.empty(int(L.sjb200_index_words(n)), dtype=torch.int32, device="cuda"))
    sharding.Comm.connect_local(comms)
    streams = [torch.cuda.Stream() for _ in range(world)]
    results = [None] * world
    barrier = threading.Barrier(world)

    def one_pass(r, name, mode):
        barrier.wait()
        t0 = time.perf_counter()
        if mode <= sj.STREAMING_FINAL:
            rc, x = comms[r].scan_stream(shards[name][r], idx[r], r == world - 1, mode, streams[r])
        else:
            rc, x = comms[r].scan_delimited(shards[name][r], idx[r], r == world - 1, mode, streams[r])
        streams[r].synchronize()
        results[r] = (rc, time.perf_counter() - t0)

    def sharded(name, mode):
        th = [threading.Thread(target=one_pass, args=(r, name, mode)) for r in range(world)]
        [t.start() for t in th]
        [t.join() for t in th]
        assert all(res[0] == 0 for res in results), (name, mode, [res[0] for res in results])
        return max(res[1] for res in results)

    rc, single = impl.create_dom_parser_implementation(cap)
    assert rc == sj.SUCCESS
    whole = {name: torch.from_numpy(np.frombuffer(doc, dtype=np.uint8).copy()).cuda() for name, doc in docs.items() if name != "ndjson"}

    def one_gpu(name, mode):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rc = single.stage1_device(whole[name], mode)
        torch.cuda.synchronize()
        assert rc == 0, (name, mode, rc)
        return time.perf_counter() - t0

    runs = [("sharded", "ndjson", sj.STREAMING_FINAL), ("sharded", "rs", 3), ("sharded", "rs", 4), ("sharded", "comma", 5), ("sharded", "comma", 6),
            ("single", "rs", 4), ("single", "comma", 6)]
    times = {k: [] for k in runs}
    for step in range(a.warmup + a.steps):
        for k in runs:  # alternated: every kind sees the same clocks and temperature
            t = sharded(k[1], k[2]) if k[0] == "sharded" else one_gpu(k[1], k[2])
            if step >= a.warmup:
                times[k].append(t)
    print(f"device (name, power limit, SM clock, max SM clock): {device_info()}")
    print(f"input: {len(rows)} NDJSON rows, {len(docs['ndjson'])} bytes as NDJSON; {world} ranks as threads on one GPU, cuts after line feeds; "
          f"median of {a.steps} passes, alternated")
    names = {2: "stream STREAMING_FINAL", 3: "JSON_SEQUENCE_PARTIAL", 4: "JSON_SEQUENCE_FINAL", 5: "COMMA_DELIMITED_PARTIAL", 6: "COMMA_DELIMITED_FINAL"}
    for k in runs:
        med = statistics.median(times[k])
        what = f"stage1_sharded_{'stream' if k[2] <= 2 else 'delimited'}" if k[0] == "sharded" else "stage1_dev (one GPU)"
        print(f"  {what:32s} {k[1]:6s} {names[k[2]]:24s} median {med * 1e3:8.3f} ms  (min {min(times[k]) * 1e3:.3f}, max {max(times[k]) * 1e3:.3f})  "
              f"{len(docs[k[1]]) / 1e9 / med:.1f} GB/s")
    single.close()
    for c in comms:
        c.close()
    for p in parsers:
        p.close()


if __name__ == "__main__":
    main()
