"""Sharded stage 1 of whitespace-separated streams (sjb200_stage1_sharded_stream*, sjb200_document_table_shard_dev): ONE
buffer cut into 2 / 4 / 8 shards, one sjb200_comm per rank, all ranks as threads of this process on one GPU
(connect_local), against stage1(whole buffer, mode) of the CPU oracle in modes 0-2 -- error code, n, kept counts, the
gathered (n+3) words, first_starts_document and the gathered per-shard document tables."""
import random
import time

import numpy as np
import pytest
import torch

import oracle_lib as O
import simdjson_b200 as sj
import stream_shards as S
from simdjson_b200 import corpus, sharding
from test_sharded_minify_utf8 import _kept, _run_ranks

pytestmark = pytest.mark.gpu

MODES = (O.REGULAR, O.STREAMING_PARTIAL, O.STREAMING_FINAL)


@pytest.fixture(scope="module")
def oracle():
    return S.Oracle()


def _stream_body(world):
    """every mode's pass in flight at once (enqueue x3, finish x3), then each rank's document table of the final pass"""
    L = sj.lib()

    def body(r, comm, p, d, stream):
        last = r == world - 1
        bufs = [torch.full((int(L.sjb200_index_words(d.numel())),), -1, dtype=torch.int32, device="cuda") for _ in MODES]
        for mode, b in zip(MODES, bufs):
            assert comm.stream_enqueue(d, b, last, mode, stream) == 0
        out = []
        for mode, b in zip(MODES, bufs):
            rc, x = comm.stream_finish()
            torch.cuda.synchronize()
            count = int(x.shard.count)
            words = b[: count + (3 if last else 0)].cpu().numpy().view(np.uint32).copy()
            table = comm.document_table(d, b, x, stream) if mode == O.STREAMING_FINAL else None
            torch.cuda.synchronize()
            out.append(dict(err=rc, n=int(x.n), kept=int(x.kept), bytes_before=int(x.bytes_before), total_bytes=int(x.total_bytes),
                            first_starts_document=int(x.first_starts_document), count=count, words=words, table=table,
                            rescanned=int(x.shard.rescanned)))
        return out
    return body


def _check_pass(oracle, buf, cuts, outs):
    buf = bytes(buf)
    a = np.frombuffer(buf, dtype=np.uint8)
    rescans = 0
    for k, mode in enumerate(MODES):
        ranks = [o[k] for o in outs]
        want = oracle.port.stage1(a, mode)
        S.check(buf, cuts, mode, want, ranks)
        rescans += sum(g["rescanned"] for g in ranks)
        if mode == O.STREAMING_FINAL and want.wrote:
            # gathered tables: local index + the ndocs prefix of the structurals before; byte + the shard's offset
            got, base = [], 0
            for g in ranks:
                for i, b in g["table"]:
                    got.append((base + int(i), (int(b) + g["bytes_before"]) & 0xFFFFFFFF))
                base += g["count"]
            starts = S.doc_starts(a, want.idx, want.n)
            assert got == [(i, int(want.idx[i])) for i in starts], (len(buf), cuts)
    return rescans


def _cases(rng):
    """(name, buffer) of the GPU cases: the CPU fold test's inputs, a few scaled up past one scan element"""
    picked = [x for x in S.inputs(rng) if not x[0].startswith(("multi", "adv")) or int(x[0][-1]) < 3]
    rows = bytes(corpus.ndjson_rows(3 << 20))
    picked.append(("ndjson_3m_cut", rows[: len(rows) - 211]))
    picked.append(("ndjson_3m_string_tail", rows[: (2 << 20)] + b'{"k": "' + b"z" * (900 << 10)))
    return picked


def test_sharded_stream_matches_whole_stage1(oracle):
    rng = random.Random(corpus.SEED ^ 0x57A)
    rescans = 0
    for name, buf in _cases(rng):
        for world in (2, 4, 8):
            sets = S.cut_sets(rng, buf, world, 2 if len(buf) > 4096 else 1)
            if len(buf) > 4096:
                sets.append(sharding.shard_cuts_at_lines(np.frombuffer(buf, dtype=np.uint8), world, window=len(buf) // (2 * world)))
            for cuts in sets:
                if any(cuts[k + 1] <= cuts[k] for k in range(world)) or oracle.shards(buf, cuts, O.STREAMING_FINAL) is None:
                    continue
                outs = _run_ranks([np.frombuffer(buf[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(world)], _stream_body(world))
                rescans += _check_pass(oracle, buf, cuts, outs)
    assert rescans > 0, "arbitrary cuts land inside strings: the second round ran"


def test_pretty_document_spanning_all_ranks(oracle):
    doc = bytes(corpus.random_json((2 << 20) + 99, pretty_bias=0.95, utf8_rate=0.1))
    for world in (2, 8):
        cuts = sharding.shard_cuts(np.frombuffer(doc, dtype=np.uint8), world)
        outs = _run_ranks([np.frombuffer(doc[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(world)], _stream_body(world))
        _check_pass(oracle, doc, cuts, outs)
        assert [o[2]["first_starts_document"] for o in outs] == [1] + [0] * (world - 1)


def test_errors_in_a_middle_shard(oracle):
    rows = bytearray(corpus.ndjson_rows(1 << 20))
    world = 4
    cuts = sharding.shard_cuts_at_lines(np.frombuffer(bytes(rows), dtype=np.uint8), world)
    mid = (cuts[1] + cuts[2]) // 2
    for what, patch in (("utf8", b"\xff"), ("control", b"\x01")):
        bad = bytearray(rows)
        q = bad.index(b'["', mid) + 2  # inside the first string of a row
        bad[q: q + 1] = patch
        outs = _run_ranks([np.frombuffer(bytes(bad[cuts[r]: cuts[r + 1]]), dtype=np.uint8) for r in range(world)], _stream_body(world))
        _check_pass(oracle, bytes(bad), cuts, outs)
        want = {"utf8": O.UTF8_ERROR, "control": O.UNESCAPED_CHARS}[what]
        assert all(o[2]["err"] == want for o in outs), what


def test_one_rank_comm_matches_stage1_dev(oracle):
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(4 << 20)
    assert rc == sj.SUCCESS
    comm = sharding.Comm(p, 0, 1)
    L = sj.lib()
    try:
        rng = random.Random(corpus.SEED ^ 0x11)
        for name, buf in _cases(rng):
            if not buf:
                continue
            d = torch.from_numpy(np.frombuffer(buf, dtype=np.uint8).copy()).cuda()
            for mode in MODES:
                rc1 = p.stage1_device(d, mode)
                n1 = p.n_structural_indexes
                w1 = p.device_index_buffer().cpu().numpy().view(np.uint32)
                b = torch.full((int(L.sjb200_index_words(len(buf))),), -1, dtype=torch.int32, device="cuda")
                rc2, x = comm.scan_stream(d, b, True, mode)
                torch.cuda.synchronize()
                want = oracle.port.stage1(np.frombuffer(buf, dtype=np.uint8), mode)
                assert rc1 == rc2 == want.err, (name, mode, rc1, rc2, want.err)
                if want.wrote:
                    w2 = b.cpu().numpy().view(np.uint32)
                    assert n1 == x.n == want.n, (name, mode)
                    assert np.array_equal(w1[: n1 + 3], w2[: n1 + 3]) and np.array_equal(w2[: n1 + 3], want.words()), (name, mode)
                else:
                    assert x.n == 0 and x.kept == 0
        for mode in range(3, 7):  # RS and comma-delimited streams are not sharded
            d = torch.from_numpy(np.frombuffer(b'{"a":1}\n[2]', dtype=np.uint8).copy()).cuda()
            b = torch.zeros(128, dtype=torch.int32, device="cuda")
            assert comm.stream_enqueue(d, b, True, mode) == sj.UNEXPECTED_ERROR
    finally:
        comm.close()
        p.close()


def test_stream_passes_in_flight_with_minify_and_utf8(oracle):
    doc = bytes(corpus.ndjson_rows(2 << 20))[: (2 << 20) - 101]
    world = 4
    cuts = sharding.shard_cuts(np.frombuffer(doc, dtype=np.uint8), world)
    L = sj.lib()
    kinds = ["stream", "minify", "validate", "stream", "minify"]
    werr, want_min = _kept(oracle.port, np.frombuffer(doc, dtype=np.uint8))

    def body(r, comm, p, d, stream):
        last = r == world - 1
        bufs = [torch.full((int(L.sjb200_index_words(d.numel())),), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
        dst = torch.empty(d.numel(), dtype=torch.uint8, device="cuda")
        js = 0
        for k in kinds:
            if k == "stream":
                rc = comm.stream_enqueue(d, bufs[js], last, O.STREAMING_FINAL, stream)
                js += 1
            elif k == "minify":
                rc = comm.minify_enqueue(d, dst, stream)
            else:
                rc = comm.validate_utf8_enqueue(d, stream)
            assert rc == 0
        rc, _ = comm.minify_finish()  # the oldest pass is a stream pass: refused, stays in flight
        assert rc == sj.UNEXPECTED_ERROR
        res = []
        js = 0
        for k in kinds:
            if k == "stream":
                rc, x = comm.stream_finish()
                torch.cuda.synchronize()
                words = bufs[js][: int(x.shard.count) + (3 if last else 0)].cpu().numpy().view(np.uint32).copy()
                js += 1
                res.append(dict(err=rc, n=int(x.n), kept=int(x.kept), bytes_before=int(x.bytes_before), total_bytes=int(x.total_bytes),
                                first_starts_document=int(x.first_starts_document), count=int(x.shard.count), words=words))
            elif k == "minify":
                rc, x = comm.minify_finish()
                res.append((rc, int(x.total_count)))
            else:
                v, _ = comm.validate_utf8_finish()
                res.append(v)
        torch.cuda.synchronize()
        return res

    outs = _run_ranks([np.frombuffer(doc[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(world)], body)
    want = oracle.port.stage1(np.frombuffer(doc, dtype=np.uint8), O.STREAMING_FINAL)
    for j, k in enumerate(kinds):
        if k == "stream":
            S.check(doc, cuts, O.STREAMING_FINAL, want, [o[j] for o in outs])
        elif k == "minify":
            assert all(o[j] == (werr, len(want_min)) for o in outs)
        else:
            assert all(o[j] == 1 for o in outs)


def test_plain_pass_against_stream_passes_fails_fast(oracle):
    doc = bytes(corpus.ndjson_rows(1 << 20))
    cuts = sharding.shard_cuts(np.frombuffer(doc, dtype=np.uint8), 2)
    L = sj.lib()

    def body(r, comm, p, d, stream):
        b = torch.zeros(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        t0 = time.monotonic()
        if r == 0:
            rc, _ = comm.scan(d, b, False, stream)
        else:
            rc, _ = comm.scan_stream(d, b, True, O.STREAMING_FINAL, stream)
        return rc, time.monotonic() - t0, p.last_cuda_error()

    outs = _run_ranks([np.frombuffer(doc[cuts[r]: cuts[r + 1]], dtype=np.uint8) for r in range(2)], body)
    for rc, dt, err in outs:
        assert rc == sj.UNEXPECTED_ERROR and "another kind" in err and dt < 5.0, (rc, dt, err)
