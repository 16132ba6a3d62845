"""Sharded minify and validate_utf8 (sjb200_minify_sharded*, sjb200_validate_utf8_sharded*): ONE buffer cut into 2 / 4 / 8
shards, one sjb200_comm per rank, all ranks as threads of this process on one GPU (connect_local), against the CPU oracle
on the whole buffer.  Also: passes of all three kinds in flight on one comm, a kind mismatch between ranks, and a
one-rank comm against the unsharded calls."""
import ctypes as C
import random
import threading

import numpy as np
import pytest
import torch

import oracle_lib as O
import simdjson_b200 as sj
from simdjson_b200 import corpus, sharding

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def port():
    return O.Port()


def _state(port, buf, state_in=0):
    """the oracle's scanner state after buf entered in state_in (bit0 escape, bit1 in string, bit2 previous byte scalar)"""
    L = port.L
    L.sjo_scan_shard.restype = C.c_uint64
    L.sjo_scan_shard.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    a = np.ascontiguousarray(buf, dtype=np.uint8)
    so = C.c_uint32(0)
    L.sjo_scan_shard(a.ctypes.data if len(a) else None, len(a), state_in, None, C.byref(so))
    return int(so.value)


def _kept(port, buf):
    """(error, kept bytes) of the oracle's minify of buf.  A buffer that ends inside a string is an error
    (UNCLOSED_STRING) but its bytes are still kept: those of buf closed by a quote, the closer removed."""
    err, out = port.minify(buf)
    if err == sj.SUCCESS:
        return err, out
    closer = (b"x" if _state(port, buf) & 1 else b"") + b'"'
    err2, out2 = port.minify(np.concatenate([buf, np.frombuffer(closer, dtype=np.uint8)]))
    assert err2 == sj.SUCCESS
    return err, out2[: len(out2) - len(closer)]


def _run_ranks(shards, body, device=0):
    """one sjb200_comm per rank, all in this process (connect_local), one thread per rank like one process per GPU;
    body(r, comm, parser, d_shard, stream) -> the rank's result"""
    world = len(shards)
    impl = sj.get_active_implementation(device)
    parsers, comms = [], []
    for r in range(world):
        rc, p = impl.create_dom_parser_implementation(max(len(shards[r]), 64))
        assert rc == sj.SUCCESS
        parsers.append(p)
        comms.append(sharding.Comm(p, r, world))
    sharding.Comm.connect_local(comms)
    out = [None] * world

    def work(r):
        try:
            torch.cuda.set_device(device)
            d = torch.from_numpy(np.array(shards[r], dtype=np.uint8)).cuda()
            out[r] = body(r, comms[r], parsers[r], d, torch.cuda.Stream())
        except Exception as e:  # noqa: BLE001
            out[r] = e

    th = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    [t.start() for t in th]
    [t.join(timeout=300) for t in th]
    assert not any(t.is_alive() for t in th), "a rank did not finish"
    for c in comms:
        c.close()
    for p in parsers:
        p.close()
    for o in out:
        if isinstance(o, Exception) or o is None:
            raise AssertionError(o)
    return out


def _minify_body(r, comm, p, d, stream):
    """two passes in flight (enqueue, enqueue, finish, finish) into one output buffer"""
    dst = torch.empty(d.numel(), dtype=torch.uint8, device="cuda")
    for _ in range(2):
        assert comm.minify_enqueue(d, dst, stream) == 0
    res = []
    for _ in range(2):
        rc, x = comm.minify_finish()
        res.append((rc, int(x.count), int(x.base), int(x.total_count), int(x.state_in), int(x.final_state), int(x.rescanned), int(x.flags_all)))
    torch.cuda.synchronize()
    return res, bytes(dst[: res[-1][1]].cpu().numpy())


def _adversarial(rng, nbytes):
    """backslash and quote runs of every parity, the cuts below land among them"""
    out = bytearray(b"[")
    while len(out) < nbytes:
        k = rng.choice([0, 1, 2, 3, 4, 31, 32, 33, 4095, 4096])
        out += b' "' + b"\\" * (2 * k) + rng.choice([b"", b'\\"', b"\\\\", b"a\\\"b"]) + b'" ,\n' + b'""' * rng.randint(0, 3) + b","
    out += b"0]"
    return np.frombuffer(bytes(out), dtype=np.uint8)


def _rows_prefix(rows, nbytes):
    """the whole NDJSON rows within the first nbytes"""
    head = bytes(rows[:nbytes])
    return head[: head.rfind(b"\n") + 1]


def _byte_cuts(rng, n, world):
    """arbitrary bytes: mid-row, mid-string, mid-UTF-8 character, right after a backslash"""
    cuts = [0] + sorted(n * k // world + rng.randint(-999, 999) for k in range(1, world)) + [n]
    return cuts


def test_sharded_minify(port):
    rng = random.Random(corpus.SEED ^ 0x313)
    ndjson = corpus.ndjson_rows(6 << 20)
    docs = [("ndjson", ndjson), ("pretty", corpus.random_json((3 << 20) + 4321, pretty_bias=0.9, utf8_rate=0.15)),
            ("adversarial", _adversarial(rng, 2 << 20)),
            ("unclosed", np.frombuffer(_rows_prefix(ndjson, 1 << 20) + b'{"k": "a \\" b \\\\ ' + b"xy z" * 17500 + b"\\", dtype=np.uint8))]  # ends in a string, escape pending
    rescans_ndjson_bytes = 0
    for name, doc in docs:
        werr, want = _kept(port, doc)
        final = _state(port, doc)
        assert (werr == sj.UNCLOSED_STRING) == (name == "unclosed") == bool(final & 2)
        for world in (2, 4, 8):
            for how, cuts in (("bytes", _byte_cuts(rng, len(doc), world)), ("lines", sharding.shard_cuts_at_lines(doc, world))):
                if any(cuts[k + 1] <= cuts[k] for k in range(world)):
                    continue
                out = _run_ranks([doc[cuts[r]: cuts[r + 1]] for r in range(world)], _minify_body)
                assert b"".join(o[1] for o in out) == want, (name, world, how)
                base = 0
                for r, (res, kept) in enumerate(out):
                    state_in = _state(port, doc[: cuts[r]])
                    for rc, count, b, total, s_in, fin, rescanned, flags_all in res:
                        assert rc == werr and count == len(kept) and b == base and total == len(want), (name, world, how, r, rc, count, b, total)
                        assert s_in == state_in and fin == final and flags_all == 0, (name, world, how, r)
                        assert rescanned == (1 if state_in & 3 else 0), (name, world, how, r, state_in)
                    base += len(kept)
                    if name == "ndjson" and how == "bytes":
                        rescans_ndjson_bytes += res[0][6]
                    if how == "lines" and name in ("ndjson", "pretty"):
                        assert res[0][6] == 0, "valid JSON cut after a line feed never needs a second scan"
    assert rescans_ndjson_bytes > 0, "arbitrary cuts of NDJSON land inside strings: the second round really ran"


def _validate_body(r, comm, p, d, stream):
    v, x = comm.validate_utf8(d, stream)
    torch.cuda.synchronize()
    return v, int(x.count), int(x.total_count), int(x.state_in), int(x.final_state), int(x.rescanned)


def test_sharded_validate_utf8(port):
    rng = random.Random(corpus.SEED ^ 0x717)
    text = corpus.random_utf8(3 << 20).copy()
    assert port.validate_utf8(text)
    for world in (2, 4, 8):
        cuts = sharding.shard_cuts(text, world)
        cases = [("valid", text)]
        r = rng.randrange(world)
        for where, at in (("start", cuts[r]), ("middle", (cuts[r] + cuts[r + 1]) // 2), ("end", cuts[r + 1] - 1 - rng.randrange(3))):
            bad = text.copy()
            bad[at] = 0xFF
            cases.append((f"shard {r} {where}", bad))
        bad = text.copy()
        bad[-1 - rng.randrange(3)] = 0xF0  # a four-byte lead in the last 3 bytes of the document: its sequence is cut short
        cases.append(("document end", bad))
        for name, buf in cases:
            want = 1 if port.validate_utf8(buf) else 0
            assert want == (1 if name == "valid" else 0), name
            out = _run_ranks([buf[cuts[k]: cuts[k + 1]] for k in range(world)], _validate_body)
            for k, (v, count, total, s_in, fin, rescanned) in enumerate(out):
                assert v == want and count == total == s_in == fin == rescanned == 0, (world, name, k, v)


def test_mixed_kinds_in_flight(port):
    """stage 1, minify and validate_utf8 passes enqueued back to back on one comm, then finished in order"""
    doc = corpus.ndjson_rows(3 << 20)
    world = 4
    cuts = sharding.shard_cuts(doc, world)
    L = sj.lib()
    werr, want_min = _kept(port, doc)
    kinds = ["stage1", "minify", "validate", "minify", "stage1", "validate"]

    def body(r, comm, p, d, stream):
        d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        dst = torch.empty(d.numel(), dtype=torch.uint8, device="cuda")
        for k in kinds:
            rc = comm.enqueue(d, d_idx, r == world - 1, stream) if k == "stage1" else comm.minify_enqueue(d, dst, stream) if k == "minify" else comm.validate_utf8_enqueue(d, stream)
            assert rc == 0
        # finishing the oldest pass with the call of another kind fails and leaves it in flight
        rc, _ = comm.minify_finish()
        assert rc == sj.UNEXPECTED_ERROR and "another kind" in p.last_cuda_error()
        res = []
        for k in kinds:
            if k == "stage1":
                rc, x = comm.finish()
            elif k == "minify":
                rc, x = comm.minify_finish()
            else:
                rc, x = comm.validate_utf8_finish()
            res.append((k, rc, int(x.count), int(x.base), int(x.total_count), int(x.rescanned)))
        torch.cuda.synchronize()
        n_idx = [x[2] for x in res if x[0] == "stage1"][-1]
        n_min = [x[2] for x in res if x[0] == "minify"][-1]
        return res, d_idx.cpu().numpy().view(np.uint32)[:n_idx].astype(np.int64) + cuts[r], bytes(dst[:n_min].cpu().numpy())

    out = _run_ranks([doc[cuts[r]: cuts[r + 1]] for r in range(world)], body)
    L2 = port.L
    L2.sjo_scan_shard.restype = C.c_uint64
    L2.sjo_scan_shard.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    widx = np.zeros(len(doc) + 1, dtype=np.uint32)
    nw = L2.sjo_scan_shard(doc.ctypes.data, len(doc), 0, widx.ctypes.data, None)
    assert np.array_equal(np.concatenate([o[1] for o in out]), widx[:nw].astype(np.int64))
    assert b"".join(o[2] for o in out) == want_min
    base = {"stage1": 0, "minify": 0}
    for r, (res, idx, kept) in enumerate(out):
        for k, rc, count, b, total, rescanned in res:
            if k == "validate":
                assert rc == 1 and count == total == 0
            else:
                assert rc == 0 and b == base[k] and total == (nw if k == "stage1" else len(want_min)), (r, k)
        base["stage1"] += len(idx)
        base["minify"] += len(kept)


def test_kind_mismatch_between_ranks(port):
    """rank 0 enqueues minify where rank 1 enqueues validate_utf8: both finishes fail instead of folding one kind's counts
    into the other's base, nothing hangs, and the comm still works for the next pass"""
    doc = corpus.ndjson_rows(1 << 20)
    cuts = sharding.shard_cuts(doc, 2)

    def body(r, comm, p, d, stream):
        dst = torch.empty(d.numel(), dtype=torch.uint8, device="cuda")
        if r == 0:
            assert comm.minify_enqueue(d, dst, stream) == 0
            rc, _ = comm.minify_finish()
        else:
            assert comm.validate_utf8_enqueue(d, stream) == 0
            rc, _ = comm.validate_utf8_finish()
        err = p.last_cuda_error()
        rc2, x = comm.minify(d, dst, stream)
        torch.cuda.synchronize()
        return rc, err, rc2, int(x.base), int(x.total_count)

    out = _run_ranks([doc[cuts[r]: cuts[r + 1]] for r in range(2)], body)
    assert out[0][0] == sj.UNEXPECTED_ERROR and out[1][0] < 0
    assert all("another kind" in o[1] for o in out)
    werr, want = _kept(port, doc)
    assert all(o[2] == werr == 0 and o[4] == len(want) for o in out) and out[0][3] == 0


def test_one_rank_comm_matches_unsharded_calls(port):
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(4 << 20)
    assert rc == sj.SUCCESS
    comm = sharding.Comm(p, 0, 1)
    try:
        rng = random.Random(corpus.SEED ^ 0x1)
        docs = [corpus.random_json((2 << 20) + 77, pretty_bias=0.9), _adversarial(rng, 300000), np.frombuffer(b'[1, "abc \\" d', dtype=np.uint8),
                corpus.random_utf8(1 << 20)]
        for doc in docs:
            d = torch.from_numpy(doc.copy()).cuda()
            dst1 = torch.zeros(len(doc), dtype=torch.uint8, device="cuda")
            dst2 = torch.zeros(len(doc), dtype=torch.uint8, device="cuda")
            rc1, n1 = p.minify_device(d, dst1)
            rc2, x = comm.minify(d, dst2)
            torch.cuda.synchronize()
            assert rc1 == rc2 and (rc1 != 0 or n1 == x.count == x.total_count) and x.base == 0 and x.rescanned == 0
            if rc1 == 0:
                assert torch.equal(dst1[:n1], dst2[:n1])
            bad = d.clone()
            bad[len(doc) // 2] = 0xFF
            for buf in (d, bad):
                v1 = p.validate_utf8_device(buf)
                v2, _ = comm.validate_utf8(buf)
                assert v1 == v2 == (1 if port.validate_utf8(buf.cpu().numpy()) else 0)
    finally:
        comm.close()
        p.close()
