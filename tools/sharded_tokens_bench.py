"""Sharded stage-2-lite on one GPU: R = 1, 2, 4 ranks as threads of this process (sjb200_comm, connect_local), each rank
one shard of the input cut after line feeds; per pass every rank runs sharded stage 1 (sjb200_stage1_sharded) and then
sjb200_tokens_sharded on its structurals.  Inputs: the 1 GiB NDJSON rows of bench.py's ndjson_1g and the 64 MiB
document of tokens_64m.  Alternated in the same session with the unsharded calls on the whole input (sjb200_stage1_dev +
sjb200_tokens_dev), so that both see the same clocks.  Prints one JSON line per (input, R): medians over the passes, the
GPU's name, power limit and SM clock beside them, and whether the gathered outputs equal sjb200_tokens_dev's.

Ranks on one GPU share its SMs, so R > 1 here measures the protocol's overhead (window polls, events, the extra
launches), not a multi-GPU speed-up.

    python tools/sharded_tokens_bench.py [--passes 10] [--ranks 1,2,4] [--inputs ndjson_1g,doc_64m]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import capi, corpus, sharding  # noqa: E402

NONE64 = (1 << 64) - 1


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    uuid = getattr(torch.cuda.get_device_properties(torch.cuda.current_device()), "uuid", None)
    sel = ["-i", "GPU-" + str(uuid)] if uuid is not None else []
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"] + sel,
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(), "note": "nvidia-smi not available"}


def make_input(name):
    if name == "ndjson_1g":
        return corpus.ndjson_rows(1 << 30)
    return corpus.random_json(64 << 20)


class Whole:
    """sjb200_stage1_dev + sjb200_tokens_dev on the whole input, outputs preallocated"""

    def __init__(self, doc):
        self.d = torch.from_numpy(doc.copy()).cuda()
        rc, self.p = sj.get_active_implementation().create_dom_parser_implementation(len(doc))
        assert rc == sj.SUCCESS
        self.cap = int(sj.lib().sjb200_string_buf_capacity(len(doc)))
        self.d_strbuf = torch.empty(self.cap, dtype=torch.uint8, device="cuda")
        self.res = capi.TokensResult()
        assert self.p.stage1_device(self.d, sj.REGULAR) == 0
        self.n = self.p.n_structural_indexes
        self.d_type = torch.empty(self.n, dtype=torch.uint8, device="cuda")
        self.d_payload = torch.empty(self.n, dtype=torch.int64, device="cuda")

    def tokens(self):
        s = torch.cuda.current_stream()
        return sj.lib().sjb200_tokens_dev(self.p._ctx, self.d.data_ptr(), self.d.numel(), self.p.device_index_buffer().data_ptr(), self.n,
                                          self.d_type.data_ptr(), self.d_payload.data_ptr(), self.d_strbuf.data_ptr(), self.cap, C.byref(self.res),
                                          C.c_void_p(s.cuda_stream))

    def step(self):
        """(stage 1 + tokens ms, tokens ms): host clock around work that ends in a synchronise; events around the tokens call"""
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        assert self.p.stage1_device(self.d, sj.REGULAR) == 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        self.rc = self.tokens()  # (the NDJSON rows carry token errors on purpose: a token error is a result here)
        assert self.rc not in (sj.CAPACITY, sj.UNEXPECTED_ERROR), self.rc
        e1.record()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, e0.elapsed_time(e1)

    def close(self):
        self.p.close()


class Sharded:
    """R ranks as threads; step() runs one pass on every rank and returns its wall time (start barrier to the last rank's
    finish) and the slowest rank's tokens time (enqueue to finish)"""

    def __init__(self, doc, world):
        self.world = world
        cuts = sharding.shard_cuts_at_lines(doc, world)
        self.cuts = cuts
        impl = sj.get_active_implementation()
        self.parsers, self.comms, self.shards, self.idx = [], [], [], []
        for r in range(world):
            rc, p = impl.create_dom_parser_implementation(max(cuts[r + 1] - cuts[r], 64))
            assert rc == sj.SUCCESS
            self.parsers.append(p)
            self.comms.append(sharding.Comm(p, r, world))
            self.shards.append(torch.from_numpy(doc[cuts[r]: cuts[r + 1]].copy()).cuda())
            self.idx.append(torch.empty(int(sj.lib().sjb200_index_words(cuts[r + 1] - cuts[r])), dtype=torch.int32, device="cuda"))
        sharding.Comm.connect_local(self.comms)
        self.go, self.done = threading.Barrier(world + 1), threading.Barrier(world + 1)
        self.out = [None] * world
        self.tok_ms = [0.0] * world
        self.stop = False
        self.error = None
        self.threads = [threading.Thread(target=self._rank, args=(r,), daemon=True) for r in range(world)]
        for t in self.threads:
            t.start()

    def _rank(self, r):
        torch.cuda.set_device(torch.cuda.current_device())
        stream = torch.cuda.Stream()
        comm, d, d_idx = self.comms[r], self.shards[r], self.idx[r]
        while True:
            self.go.wait()
            if self.stop:
                return
            try:
                rc, x = comm.scan(d, d_idx, r == self.world - 1, stream)
                assert rc == 0, rc
                t0 = time.perf_counter()
                rc, res, t, p, sb = comm.tokens(d, d_idx, int(x.count), int(x.state_in), None, stream)
                self.tok_ms[r] = (time.perf_counter() - t0) * 1e3
                assert rc not in (sj.CAPACITY, sj.UNEXPECTED_ERROR), (rc, comm.parser.last_cuda_error())
                self.out[r] = (rc, res, t, p, sb)
            except Exception as e:  # noqa: BLE001
                self.error = e
            self.done.wait()

    def step(self):
        t0 = time.perf_counter()
        self.go.wait()
        self.done.wait()
        if self.error:
            raise self.error
        return (time.perf_counter() - t0) * 1e3, max(self.tok_ms)

    def matches(self, whole):
        """the gathered, rebased outputs of the last pass == sjb200_tokens_dev on the whole input"""
        types, pays, sbs = [], [], []
        fe = NONE64 if whole.res.first_error_index == 0xFFFFFFFF else int(whole.res.first_error_index)
        for rc, res, t, p, sb in self.out:
            if rc != whole.rc or res.first_error_index != fe:
                return False
            p = p.clone()
            p[t == ord('"')] += int(res.string_base)
            p[t == ord("d")] += int(res.bytes_before)
            types.append(t); pays.append(p); sbs.append(sb[: int(res.string_bytes)])
        n, sbytes = whole.n, int(whole.res.string_bytes)
        return (torch.equal(torch.cat(types), whole.d_type[:n]) and torch.equal(torch.cat(pays), whole.d_payload[:n])
                and torch.equal(torch.cat(sbs), whole.d_strbuf[:sbytes]))

    def close(self):
        self.stop = True
        self.go.wait()
        for t in self.threads:
            t.join()
        for c in self.comms:
            c.close()
        for p in self.parsers:
            p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ranks", default="1,2,4")
    ap.add_argument("--inputs", default="ndjson_1g,doc_64m")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sharded_tokens_bench needs a GPU")
    for name in args.inputs.split(","):
        doc = make_input(name)
        whole = Whole(doc)
        for world in [int(x) for x in args.ranks.split(",")]:
            sh = Sharded(doc, world)
            info_before = gpu_info()
            w_all, w_tok, s_all, s_tok = [], [], [], []
            for it in range(args.warmup + args.passes):
                a, b = whole.step()
                c, d = sh.step()
                if it >= args.warmup:
                    w_all.append(a); w_tok.append(b); s_all.append(c); s_tok.append(d)
            ok = sh.matches(whole)
            polls = sum(p.get_stat("xchg_polls") for p in sh.parsers)
            line = {"input": name, "bytes": len(doc), "ranks": world, "cuts": sh.cuts, "passes": args.passes,
                    "sharded_stage1_tokens_ms": round(statistics.median(s_all), 3), "sharded_tokens_ms": round(statistics.median(s_tok), 3),
                    "whole_stage1_tokens_ms": round(statistics.median(w_all), 3), "whole_tokens_dev_ms": round(statistics.median(w_tok), 3),
                    "spread_sharded_ms": [round(min(s_all), 3), round(max(s_all), 3)], "spread_whole_ms": [round(min(w_all), 3), round(max(w_all), 3)],
                    "window_polls_all_ranks": polls, "error": int(whole.rc), "outputs_match_tokens_dev": bool(ok),
                    "timing": "host clock from the start of the pass to the last rank's finish (sharded) / to a synchronise (whole); "
                              "whole_tokens_dev_ms: CUDA events around sjb200_tokens_dev; sharded_tokens_ms: the slowest rank's tokens enqueue + finish",
                    "ranks_are": "threads of one process on ONE GPU (they share its SMs)",
                    "gpu": info_before, "gpu_after": gpu_info()}
            print(json.dumps(line), flush=True)
            sh.close()
        whole.close()
        del whole
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
