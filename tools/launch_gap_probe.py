"""Where the time between two stage-1 launches goes (tuning aid).

    python tools/launch_gap_probe.py [--steps 100] [--reps 3] [--root CHECKOUT] [--out FILE]

The bench's workload: `steps` documents of 64 MiB through sjb200_stage1_dev_batch, 4 distinct inputs and 4 index arrays
rotating, so every launch scans 4 documents.  With option launch_stamps each launch records the globaltimer at its
first CTA's entry and at its last CTA's exit; from them, per launch, the gap to the previous launch's exit (negative:
the launches overlap by that much) and the launch's own span.  Run with pdl 0 (plain launches, nothing queued between
them) and pdl 1 (each launch may start while the previous one runs).  --root: the package of another built checkout;
one without sjb200_get_launch_stamps (an older one, whose table copies sit between the launches) reports the step time
only.  Prints one JSON line per configuration."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

DOC_BYTES = 64 << 20
ROTATE = 4


def stats(a):
    a = np.asarray(a, dtype=np.float64)
    return {"median": round(float(np.median(a)), 2), "min": round(float(a.min()), 2), "max": round(float(a.max()), 2)} if len(a) else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import simdjson_b200 as sj
    from simdjson_b200 import corpus
    L = sj.lib()
    has_stamps = hasattr(L, "sjb200_get_launch_stamps")
    if has_stamps:
        L.sjb200_get_launch_stamps.restype = C.c_long
        L.sjb200_get_launch_stamps.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    rc, parser = sj.get_active_implementation().create_dom_parser_implementation(DOC_BYTES)
    assert rc == sj.SUCCESS, sj.ERROR_NAMES.get(rc, rc)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    docs = [torch.from_numpy(corpus.random_json(DOC_BYTES, seed=corpus.SEED + 7919 * k).copy()).to(dev) for k in range(ROTATE)]
    words = L.sjb200_index_words(DOC_BYTES)
    idxs = [torch.empty(words, dtype=torch.int32, device=dev) for _ in range(ROTATE)]
    bufs = [docs[i % ROTATE] for i in range(args.steps)]
    outs = [idxs[i % ROTATE] for i in range(args.steps)]
    lines = []
    for pdl in ((0, 1) if has_stamps else (None,)):
        if pdl is not None:
            parser.set_option("pdl", pdl)
            parser.set_option("launch_stamps", 1)
        step_us, gaps, spans = [], [], []
        for rep in range(args.reps + 1):  # the first round warms up
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(stream)
            res = parser.stage1_device_batch(bufs, outs, sj.REGULAR, stream=stream)
            e1.record(stream)
            torch.cuda.synchronize()
            assert all(err == sj.SUCCESS for err, _ in res)
            if rep == 0:
                continue
            step_us.append(e0.elapsed_time(e1) * 1e3 / args.steps)
            if has_stamps:
                st = np.zeros((args.steps, 2), dtype=np.uint64)
                n = L.sjb200_get_launch_stamps(parser._ctx, st.ctypes.data, args.steps)
                t = st[:n].astype(np.int64)
                spans += list((t[:, 1] - t[:, 0]) / 1e3)
                gaps += list((t[1:, 0] - t[:-1, 1]) / 1e3)
        line = {"root": args.root, "pdl": pdl, "steps": args.steps, "documents_per_launch": ROTATE, "step_us": stats(step_us)}
        if has_stamps:
            line["launch_span_us"] = stats(spans)  # first CTA in -> last CTA out
            line["gap_us"] = stats(gaps)  # next launch's first CTA in - this launch's last CTA out (< 0: overlap)
            line["overlap_us"] = stats([max(0.0, -g) for g in gaps])
        print(json.dumps(line), flush=True)
        lines.append(line)
    parser.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
