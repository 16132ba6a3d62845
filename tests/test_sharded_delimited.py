"""Sharded stage 1 of RS-delimited and comma-delimited streams (sjb200_stage1_sharded_delimited*): ONE buffer cut into
2 / 4 / 8 shards, one sjb200_comm per rank, all ranks as threads of this process on one GPU (connect_local), against
stage1(whole buffer, mode) of the CPU oracle in modes 3-6 -- error code, n, kept and filtered counts, the gathered
(n+3) words, first_starts_document and the gathered per-shard document tables."""
import random
import time

import numpy as np
import pytest
import torch

import delimited_shards as D
import oracle_lib as O
import simdjson_b200 as sj
import stream_shards as S
from simdjson_b200 import corpus, sharding
from test_sharded_minify_utf8 import _kept, _run_ranks

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle():
    return S.Oracle()


def _result(rc, x, b, with_words=True):
    filtered = int(x.filtered)
    return dict(err=rc, n=int(x.stream.n), kept=int(x.stream.kept), bytes_before=int(x.stream.bytes_before), total_bytes=int(x.stream.total_bytes),
                first_starts_document=int(x.stream.first_starts_document), filtered=filtered, filtered_before=int(x.filtered_before),
                words=b[:filtered].cpu().numpy().view(np.uint32).copy() if with_words else None, tail=[int(t) for t in x.tail],
                rescanned=int(x.stream.shard.rescanned))


def _delimited_body(world):
    """every delimited mode's pass in flight at once (enqueue x4, finish x4), then each rank's document table"""
    L = sj.lib()

    def body(r, comm, p, d, stream):
        last = r == world - 1
        bufs = [torch.full((int(L.sjb200_index_words(d.numel())),), -1, dtype=torch.int32, device="cuda") for _ in D.MODES]
        for mode, b in zip(D.MODES, bufs):
            assert comm.delimited_enqueue(d, b, last, mode, stream) == 0
        out = []
        for mode, b in zip(D.MODES, bufs):
            rc, x = comm.delimited_finish()
            torch.cuda.synchronize()
            g = _result(rc, x, b)
            g["table"] = comm.document_table(d, b, x.stream, stream)
            torch.cuda.synchronize()
            out.append(g)
        return out
    return body


def _check_pass(oracle, buf, cuts, outs):
    buf = bytes(buf)
    a = np.frombuffer(buf, dtype=np.uint8)
    rescans = 0
    for k, mode in enumerate(D.MODES):
        ranks = [o[k] for o in outs]
        want = oracle.port.stage1(a, mode)
        D.check(buf, cuts, mode, want, ranks)
        rescans += sum(g["rescanned"] for g in ranks)
        if want.wrote:
            # gathered tables: local index + the filtered entries before; byte + the shard's offset
            got = []
            for g in ranks:
                for i, b in g["table"]:
                    got.append((g["filtered_before"] + int(i), (int(b) + g["bytes_before"]) & 0xFFFFFFFF))
            starts = S.doc_starts(a, want.idx, want.n)
            assert got == [(i, int(want.idx[i])) for i in starts], (len(buf), cuts, mode)
    return rescans


def _cases(rng):
    """(name, buffer): a few of the CPU fold test's inputs, the special cases, and streams past one scan element"""
    picked = [(n, b) for n, b, _ in D.inputs(rng, nfuzz=3)]
    rows = [r for r in bytes(corpus.ndjson_rows(3 << 20)).split(b"\n") if r]
    picked.append(("rs_3m", b"".join(b"\x1e" + r + b"\n" for r in rows)))
    picked.append(("comma_3m_cut", b",\n".join(rows)[:-211]))
    picked.append(("rs_3m_string_tail", b"".join(b"\x1e" + r + b"\n" for r in rows[: len(rows) // 2]) + b'\x1e{"k": "' + b"z, \x1e " * (300 << 10)))
    return picked


def test_sharded_delimited_matches_whole_stage1(oracle):
    rng = random.Random(corpus.SEED ^ 0xDE5)
    rescans = 0
    for name, buf in _cases(rng):
        for world in (2, 4, 8):
            sets = D.cut_sets(rng, buf, world, 2 if len(buf) > 4096 else 1)
            if len(buf) > 4096:
                sets.append(sharding.shard_cuts_at_lines(np.frombuffer(buf, dtype=np.uint8), world, window=len(buf) // (2 * world)))
            for cuts in sets:
                if any(cuts[k + 1] <= cuts[k] for k in range(world)) or oracle.shards(buf, cuts, O.JSON_SEQUENCE_FINAL) is None:
                    continue
                outs = _run_ranks([np.frombuffer(buf[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(world)], _delimited_body(world))
                rescans += _check_pass(oracle, buf, cuts, outs)
    assert rescans > 0, "arbitrary cuts land inside strings: the second round ran"


def test_one_rank_comm_matches_stage1_dev(oracle):
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(4 << 20)
    assert rc == sj.SUCCESS
    comm = sharding.Comm(p, 0, 1)
    L = sj.lib()
    try:
        rng = random.Random(corpus.SEED ^ 0x12)
        for name, buf in _cases(rng):
            d = torch.from_numpy(np.frombuffer(buf, dtype=np.uint8).copy()).cuda()
            for mode in D.MODES:
                rc1 = p.stage1_device(d, mode)
                n1 = p.n_structural_indexes
                w1 = p.device_index_buffer().cpu().numpy().view(np.uint32)
                b = torch.full((int(L.sjb200_index_words(len(buf))),), -1, dtype=torch.int32, device="cuda")
                rc2, x = comm.scan_delimited(d, b, True, mode)
                torch.cuda.synchronize()
                want = oracle.port.stage1(np.frombuffer(buf, dtype=np.uint8), mode)
                assert rc1 == rc2 == want.err, (name, mode, rc1, rc2, want.err)
                if want.wrote:
                    n = int(x.stream.n)
                    got = np.concatenate([b[: int(x.stream.kept)].cpu().numpy().view(np.uint32), np.array(list(x.tail), dtype=np.uint32)])
                    assert n1 == n == want.n, (name, mode)
                    assert np.array_equal(w1[: n1 + 3], got[: n + 3]) and np.array_equal(got[: n + 3], want.words()), (name, mode)
                else:
                    assert x.stream.n == 0 and x.stream.kept == 0
        for mode in range(0, 3):  # whitespace-separated streams go through sjb200_stage1_sharded_stream
            d = torch.from_numpy(np.frombuffer(b'{"a":1}\n[2]', dtype=np.uint8).copy()).cuda()
            b = torch.zeros(128, dtype=torch.int32, device="cuda")
            assert comm.delimited_enqueue(d, b, True, mode) == sj.UNEXPECTED_ERROR
    finally:
        comm.close()
        p.close()


def test_delimited_passes_in_flight_with_stream_passes_and_minify(oracle):
    rows = [r for r in bytes(corpus.ndjson_rows(2 << 20)).split(b"\n") if r]
    doc = b"".join(b"\x1e" + r + b"\n" for r in rows)[: (2 << 20) - 77]
    world = 4
    cuts = sharding.shard_cuts(np.frombuffer(doc, dtype=np.uint8), world)
    L = sj.lib()
    kinds = [("delim", O.JSON_SEQUENCE_FINAL), ("stream", O.STREAMING_FINAL), ("minify", None), ("delim", O.COMMA_DELIMITED_PARTIAL),
             ("stream", O.REGULAR), ("delim", O.JSON_SEQUENCE_PARTIAL)]
    werr, want_min = _kept(oracle.port, np.frombuffer(doc, dtype=np.uint8))

    def body(r, comm, p, d, stream):
        last = r == world - 1
        bufs = [torch.full((int(L.sjb200_index_words(d.numel())),), -1, dtype=torch.int32, device="cuda") for _ in kinds]
        dst = torch.empty(d.numel(), dtype=torch.uint8, device="cuda")
        for (k, mode), b in zip(kinds, bufs):
            rc = {"delim": lambda: comm.delimited_enqueue(d, b, last, mode, stream), "stream": lambda: comm.stream_enqueue(d, b, last, mode, stream),
                  "minify": lambda: comm.minify_enqueue(d, dst, stream)}[k]()
            assert rc == 0
        rc, _ = comm.stream_finish()  # the oldest pass is a delimited pass: refused, stays in flight
        assert rc == sj.UNEXPECTED_ERROR
        res = []
        for (k, mode), b in zip(kinds, bufs):
            if k == "delim":
                rc, x = comm.delimited_finish()
                torch.cuda.synchronize()
                res.append(_result(rc, x, b))
            elif k == "stream":
                rc, x = comm.stream_finish()
                torch.cuda.synchronize()
                words = b[: int(x.shard.count) + (3 if last else 0)].cpu().numpy().view(np.uint32).copy()
                res.append(dict(err=rc, n=int(x.n), kept=int(x.kept), bytes_before=int(x.bytes_before), total_bytes=int(x.total_bytes),
                                first_starts_document=int(x.first_starts_document), count=int(x.shard.count), words=words))
            else:
                rc, x = comm.minify_finish()
                res.append((rc, int(x.total_count)))
        torch.cuda.synchronize()
        return res

    outs = _run_ranks([np.frombuffer(doc[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(world)], body)
    a = np.frombuffer(doc, dtype=np.uint8)
    for j, (k, mode) in enumerate(kinds):
        if k == "delim":
            D.check(doc, cuts, mode, oracle.port.stage1(a, mode), [o[j] for o in outs])
        elif k == "stream":
            S.check(doc, cuts, mode, oracle.port.stage1(a, mode), [o[j] for o in outs])
        else:
            assert all(o[j] == (werr, len(want_min)) for o in outs)


@pytest.mark.parametrize("other", ["plain", "stream", "minify", "validate"])
def test_other_kinds_against_delimited_passes_fail_fast(oracle, other):
    doc = b"".join(b"\x1e" + r + b"\n" for r in bytes(corpus.ndjson_rows(1 << 20)).split(b"\n") if r)
    cuts = sharding.shard_cuts(np.frombuffer(doc, dtype=np.uint8), 2)
    L = sj.lib()

    def body(r, comm, p, d, stream):
        b = torch.zeros(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        t0 = time.monotonic()
        if r == 0:
            if other == "plain":
                rc, _ = comm.scan(d, b, False, stream)
            elif other == "stream":
                rc, _ = comm.scan_stream(d, b, False, O.STREAMING_FINAL, stream)
            elif other == "minify":
                rc, _ = comm.minify(d, torch.empty(d.numel(), dtype=torch.uint8, device="cuda"), stream)
            else:
                v, _ = comm.validate_utf8(d, stream)
                rc = sj.UNEXPECTED_ERROR if v < 0 else v
        else:
            rc, _ = comm.scan_delimited(d, b, True, O.JSON_SEQUENCE_FINAL, stream)
        return rc, time.monotonic() - t0, p.last_cuda_error()

    outs = _run_ranks([np.frombuffer(doc[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(2)], body)
    for rc, dt, err in outs:
        assert rc == sj.UNEXPECTED_ERROR and "another kind" in err and dt < 5.0, (rc, dt, err)
