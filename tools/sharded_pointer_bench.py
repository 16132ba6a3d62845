"""Sharded JSON Pointer lookup on one GPU: R = 1, 2, 4 ranks as threads of this process (sjb200_comm, connect_local),
each rank one shard of the input cut after line feeds.  Every rank runs sharded stage 1 (streaming-final for the NDJSON
rows, plain for the single document), its document table and sharded tokens once; then each pass times
sjb200_at_pointer_sharded on every rank (wall clock, from a common start to the last rank's return), alternated in the
same session with sjb200_at_pointer_dev on the gathered arrays (CUDA events), so that both see the same clocks.  Before
the timed passes every rank runs 64 untimed ones, so that each window slot has its scratch.  Inputs: 1 GiB of twitter
status rows with 4 pointers (table mode), and the 64 MiB document of tokens_64m (whole mode) with its first, middle and
last root element -- the last one's walk crosses every cut.  Prints one JSON line per (input, R): medians over the
passes, with the GPU's name, power limit and SM clock, and whether the gathered results equal the unsharded call's.

Ranks on one GPU share its SMs, so R > 1 here measures the protocol's overhead (the edge round, one count round per step
of the walks, window polls, the extra launches), not a multi-GPU speed-up.  In whole mode a walk crosses the ranks one
after the other, so the sharded call is expected to be no faster than the unsharded one: what it saves is the gather.

    python tools/sharded_pointer_bench.py [--passes 10] [--ranks 1,2,4] [--inputs twitter_1g,doc_64m]
"""
import argparse
import ctypes as C
import json
import lzma
import os
import statistics
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import simdjson_b200 as sj  # noqa: E402
from simdjson_b200 import capi, corpus, sharding  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sharded_tokens_bench import gpu_info  # noqa: E402

WARM = 64  # kXchgSteps: the window slots a comm cycles through
TWITTER_POINTERS = ["/id", "/user/screen_name", "/entities/hashtags/0/text", "/retweet_count"]


def make_input(name):
    if name == "twitter_1g":
        with lzma.open(os.path.join(ROOT, "tests", "golden", "jsonexamples", "twitter.json.xz")) as f:
            rows = [json.dumps(s, ensure_ascii=False).encode() for s in json.load(f)["statuses"]]
        block = b"\n".join(rows) + b"\n"
        return (block * ((1 << 30) // len(block) + 1))[: 1 << 30].rsplit(b"\n", 1)[0] + b"\n"
    return bytes(corpus.random_json(64 << 20))


def root_pointers(types):
    """the first, middle and last element of the root array of one document's token types"""
    assert types[0] == ord("["), "the generator's root is an array"
    t = torch.from_numpy(types).cuda()
    delta = (t == ord("{")).int() + (t == ord("[")).int() - (t == ord("}")).int() - (t == ord("]")).int()
    depth = torch.cumsum(delta, 0) - delta  # depth entering each structural
    count = int(((depth == 1) & (t != ord(",")) & (t != ord("]"))).sum())
    return [f"/{k}" for k in (0, count // 2, count - 1)]


def cuts_at_lines(doc, world):
    return sharding.shard_cuts_at_lines(doc, world, window=max(1, len(doc) // (2 * world)))


def run(name, doc, world, passes):
    whole = name != "twitter_1g"
    mode = None if whole else capi.STREAMING_FINAL
    L = sj.lib()
    cuts = cuts_at_lines(doc, world)
    impl = sj.get_active_implementation()
    parsers, comms = [], []
    for r in range(world):
        rc, p = impl.create_dom_parser_implementation(max(cuts[r + 1] - cuts[r], 64))
        assert rc == sj.SUCCESS
        parsers.append(p)
        comms.append(sharding.Comm(p, r, world))
    sharding.Comm.connect_local(comms)
    gate = threading.Barrier(world + 1)
    times, outs, errs = [[] for _ in range(world)], [None] * world, []
    pointers = [None]

    def work(r):
        try:
            comm, stream = comms[r], torch.cuda.Stream()
            d = torch.from_numpy(doc[cuts[r]: cuts[r + 1]].copy()).cuda()
            d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
            last = r == world - 1
            table = None
            if mode is None:
                rc, x = comm.scan(d, d_idx, last, stream)
                n, shard_len = int(x.count), d.numel()
            else:
                rc, x = comm.scan_stream(d, d_idx, last, mode, stream)
                n, shard_len = int(x.kept), (int(x.total_bytes - x.bytes_before) if last else d.numel())
                table = comm.document_table(d, d_idx, x, stream)
            assert rc == 0
            _, y, t, pay, sb = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)
            del d_idx, d
            torch.cuda.synchronize()
            outs[r] = [None, t, pay, n, table, sb[: int(y.string_bytes)], int(y.string_base)]
            gate.wait()  # the tokens are out; then the pointers (whole mode: from the gathered types)
            gate.wait()
            ps = pointers[0]
            enc = [q.encode() for q in ps]
            bufs = [C.create_string_buffer(e, len(e)) for e in enc]
            ptrs = (C.c_void_p * len(enc))(*[C.addressof(b) for b in bufs])
            lens = (C.c_size_t * len(enc))(*[len(e) for e in enc])
            nd = 0 if whole or table is None else len(table)
            d_docs = torch.from_numpy(np.ascontiguousarray(table.astype(np.uint32)).view(np.int32).reshape(-1)).cuda() if nd else None
            k = 1 if whole else nd
            d_out = torch.empty(max(k * len(enc), 1) * 2, dtype=torch.int64, device="cuda")
            res = capi.ShardedPointerSummary()

            def call():
                return L.sjb200_at_pointer_sharded(comm._h, t.data_ptr() if n else None, pay.data_ptr() if n else None, n, sb.data_ptr(), int(y.string_bytes),
                                                   int(whole), d_docs.data_ptr() if nd else None, nd, ptrs, lens, len(enc), d_out.data_ptr(), res,
                                                   stream.cuda_stream)
            for _ in range(WARM):  # every window slot's scratch is grow-only and allocated on the slot's first pass
                assert call() == 0
            torch.cuda.synchronize()
            gate.wait()
            for _ in range(passes + 1):
                gate.wait()
                t0 = time.perf_counter()
                rc = call()
                times[r].append(time.perf_counter() - t0)
                assert rc == 0, rc
                gate.wait()
            k = 1 if whole and r == 0 else (0 if whole else nd)
            o = d_out[: 2 * k * len(enc)].cpu().numpy().view(np.uint64).reshape(len(enc), k, 2)
            outs[r][0] = (rc, res, (o[:, :, 0] & 0xFFFFFFFF).astype(np.uint32).view(np.int32), o[:, :, 1].copy())
        except Exception as e:  # noqa: BLE001
            errs.append(e)
            gate.abort()

    th = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    [t.start() for t in th]
    ref_ms = []
    try:
        gate.wait()
        t_all, pay_all, sb_all, p, docs, nd = gathered(outs, impl)
        pointers[0] = root_pointers(t_all.cpu().numpy()) if whole else TWITTER_POINTERS
        gate.wait()
        gate.wait()  # every rank has warmed its window slots
        for k in range(passes + 1):
            gate.wait()
            gate.wait()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            e, i = p.at_pointer_device(pointers[0], t_all, pay_all, sb_all, sb_all.numel(), docs, nd)
            e1.record()
            torch.cuda.synchronize()
            if k:
                ref_ms.append(e0.elapsed_time(e1))
    except threading.BrokenBarrierError:
        pass
    [t.join() for t in th]
    if errs:
        raise errs[0]
    got_e = np.concatenate([o[0][2] for o in (outs[:1] if whole else outs)], axis=1)
    got_i = np.concatenate([o[0][3] for o in (outs[:1] if whole else outs)], axis=1)
    wi = i.cpu().numpy().view(np.uint32)
    want_i = np.where(wi == 0xFFFFFFFF, np.uint64((1 << 64) - 1), wi.astype(np.uint64))
    same = bool(np.array_equal(got_e, e.cpu().numpy()) and np.array_equal(got_i, want_i))
    assert same, "the sharded results differ from sjb200_at_pointer_dev on the gathered arrays"
    sharded_ms = [1e3 * max(times[r][k] for r in range(world)) for k in range(1, passes + 1)]
    s0 = outs[0][0][1]
    for c in comms:
        c.close()
    for q in parsers + [p]:
        q.close()
    return {"input": name, "ranks": world, "mode": "whole" if whole else "table", "structurals": int(t_all.numel()), "documents": int(s0.ndocs),
            "pointers": pointers[0], "rounds": int(s0.rounds), "sharded_ms_median": statistics.median(sharded_ms),
            "unsharded_ms_median": statistics.median(ref_ms), "passes": passes, "equal": same}


def gathered(outs, impl):
    """the concatenation of the ranks' tokens (string payloads rebased), string buffers and tables, and a parser for the
    unsharded call on them"""
    t_all = torch.cat([o[1] for o in outs])
    pays = []
    for o in outs:
        q = o[2].clone()
        q[o[1] == ord('"')] += o[6]
        pays.append(q)
    pay_all = torch.cat(pays)
    sb_all = torch.cat([o[5] for o in outs])
    starts, before = [], 0
    for o in outs:
        if o[4] is not None:
            starts.append(o[4][:, 0] + before)
        before += o[3]
    rc, p = impl.create_dom_parser_implementation(1 << 16)
    docs = None
    if starts:
        s = np.concatenate(starts).astype(np.uint32)
        docs = torch.from_numpy(np.stack([s, np.zeros_like(s)], 1).reshape(-1).view(np.int32).copy()).cuda()
    return t_all, pay_all, sb_all, p, docs, None if docs is None else docs.numel() // 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--ranks", default="1,2,4")
    ap.add_argument("--inputs", default="twitter_1g,doc_64m")
    a = ap.parse_args()
    info = gpu_info()
    for name in a.inputs.split(","):
        doc = np.frombuffer(make_input(name), dtype=np.uint8)
        for world in [int(x) for x in a.ranks.split(",")]:
            row = run(name, doc, world, a.passes)
            row.update(gpu=info)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
