"""Sharded stage-2-lite (sjb200_tokens_sharded*): ONE document cut into 2 / 4 / 8 shards at clean cuts, stage 1 sharded
(the plain, streaming and comma-delimited passes), then tokens on every rank's structurals; all ranks as threads of this
process on one GPU (connect_local).  The gathered outputs -- types, payloads rebased by string_base / bytes_before, the
ranks' parts of the string buffer -- must equal the oracle's and sjb200_tokens_dev's on the whole document, and every
rank must return the same verdict.  Also: errors, capacity, dirty cuts, empty shards, passes of other kinds in flight,
a kind mismatch and a one-rank comm."""
import random
import time

import numpy as np
import pytest
import torch

import oracle_lib as O
import simdjson_b200 as sj
import token_fuzz as TF
from simdjson_b200 import capi, corpus, sharding
from test_sharded_minify_utf8 import _run_ranks
from test_tokens_shards_emul import _fuzz_docs

pytestmark = pytest.mark.gpu

NONE64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def port():
    return O.Port()


def _fields(rc, x, t, p, sb):
    f = {name: int(getattr(x, name)) for name, _ in capi.ShardedTokensResult._fields_}
    f["rc"] = rc
    if t is not None:
        f["types"] = t.cpu().numpy().copy()
        f["pay"] = p.cpu().numpy().view(np.uint64).copy()
        f["sb"] = bytes(sb[: min(f["string_bytes"], sb.numel())].cpu().numpy())
    return f


def _tokens(comm, d, d_idx, n, state_in, stream, cap=None):
    rc, x, t, p, sb = comm.tokens(d, d_idx, n, state_in, cap, stream)
    torch.cuda.synchronize()
    return _fields(rc, x, t, p, sb)


def _stage1_body(caps=None):
    """sjb200_stage1_sharded, then tokens over its count structurals"""
    def body(r, comm, p, d, stream):
        d_idx = torch.empty(int(sj.lib().sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        rc, x = comm.scan(d, d_idx, r == comm.world - 1, stream)
        assert rc == 0, rc
        f = _tokens(comm, d, d_idx, int(x.count), int(x.state_in), stream, None if caps is None else caps[r])
        f["stage1_state_in"] = int(x.state_in)
        return f
    return body


def _whole(port, doc, idx, n):
    """the oracle's tokens of the whole document, checked against sjb200_tokens_dev on it"""
    want = port.tokens(doc, idx, n)
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(max(len(doc), 64))
    assert rc == sj.SUCCESS
    try:
        d = torch.from_numpy(np.frombuffer(bytes(doc), dtype=np.uint8).copy()).cuda()
        d_idx = torch.from_numpy(np.ascontiguousarray(idx[: max(n, 1)], dtype=np.uint32).view(np.int32)).cuda()
        res, t, pay, sb = p.tokens_device(d, d_idx, n)
        torch.cuda.synchronize()
        assert res.error == want[0] and res.first_error_index == want[6] and res.n_strings == want[5] and res.string_bytes == want[4]
        assert bytes(t.cpu().numpy()) == bytes(want[1]) and np.array_equal(pay.cpu().numpy().view(np.uint64), want[2])
        assert bytes(sb[: res.string_bytes].cpu().numpy()) == bytes(want[3])
    finally:
        p.close()
    return want


def _check(outs, want, what):
    """every rank the whole document's verdict; the gathered, rebased outputs the whole document's"""
    err, types, pay, sb, sl, ns, fe = want
    tokens = strings = string_bytes = 0
    got_t, got_p, got_s = [], [], []
    for r, o in enumerate(outs):
        assert o["rc"] == o["error"] == err and o["dirty_cuts"] == 0 and o["short_ranks"] == 0, (what, r, o["rc"], err)
        assert o["first_error_index"] == (NONE64 if fe == 0xFFFFFFFF else fe), (what, r, o["first_error_index"], fe)
        assert o["total_strings"] == ns and o["total_string_bytes"] == sl, (what, r)
        assert (o["tokens_before"], o["strings_before"], o["string_base"]) == (tokens, strings, string_bytes), (what, r)
        p = o["pay"].copy()
        p[o["types"] == ord('"')] += np.uint64(o["string_base"])
        p[o["types"] == ord("d")] += np.uint64(o["bytes_before"])
        got_t.append(bytes(o["types"])); got_p.append(p); got_s.append(o["sb"])
        tokens += len(o["types"]); strings += o["n_strings"]; string_bytes += o["string_bytes"]
    assert b"".join(got_t) == bytes(types), what
    assert np.array_equal(np.concatenate(got_p), pay), what
    assert b"".join(got_s) == bytes(sb), what


def _row(rng, k):
    """one record without a token error: strings with escapes, integers, floats, atoms"""
    s1 = TF.string_body(rng, bad_rate=0.0)[0]
    s2 = TF.string_body(rng, bad_rate=0.0, maxlen=300)[0]
    return (b'{"id": %d, "name": "%s", "v": [%d.%d, true, null, -%d], "s": "%s", "t": false}'
            % (k, s1, rng.randrange(10 ** 6), rng.randrange(100), rng.randrange(10 ** 12), s2))


def _array_doc(rng, nrows, bad_rows=()):
    """a JSON array of records, one per line; only the rows in bad_rows carry a token error"""
    rows = [_row(rng, k) for k in range(nrows)]
    for k in bad_rows:
        rows[k] = rows[k][:-1] + b', "bad": ' + rng.choice([b"tru", b"nul", b"-x", b"01", b'"\\q"']) + b"}"
    return b"[\n" + b",\n".join(rows) + b"\n]\n", rows


def test_stage1_sharded_then_tokens(port):
    rng = random.Random(corpus.SEED ^ 0x70E)
    doc, rows = _array_doc(rng, 12000)
    docs = [("rows", doc)] + [(f"fuzz{i}", d) for i, d in enumerate(_fuzz_docs(rng, 3))]
    for name, d in docs:
        a = np.frombuffer(d, dtype=np.uint8)
        w = port.stage1(a)
        assert w.err == 0
        want = _whole(port, a, w.idx, w.n)
        assert want[0] == 0 if name == "rows" else want[0] not in (1,)
        for world in (2, 4, 8):
            cuts = sharding.shard_cuts_at_lines(a, world, window=len(a) // (2 * world))
            if any(cuts[k + 1] <= cuts[k] for k in range(world)):
                continue
            outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(world)], _stage1_body())
            assert all(o["stage1_state_in"] == 0 for o in outs)
            for r, o in enumerate(outs):
                assert o["bytes_before"] == cuts[r]
            _check(outs, want, (name, world))


def test_token_errors_fold_to_the_first(port):
    """errors in several ranks, and in the last rank only: every rank returns the code and global index of the first"""
    rng = random.Random(corpus.SEED ^ 0xBAD)
    for world in (2, 4, 8):
        for bad in ((7, 5000, 9000, 11990), (11900,), (3000, 3001)):
            doc, _ = _array_doc(rng, 12000, bad)
            a = np.frombuffer(doc, dtype=np.uint8)
            w = port.stage1(a)
            want = _whole(port, a, w.idx, w.n)
            assert want[0] not in (0, 1)
            cuts = sharding.shard_cuts_at_lines(a, world, window=len(a) // (2 * world))
            outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(world)], _stage1_body())
            _check(outs, want, (world, bad))


def test_capacity(port):
    """one rank short of string buffer: CAPACITY on every rank with its bit, the others' outputs as usual; a token error
    together with a short rank: the token error"""
    rng = random.Random(corpus.SEED ^ 0xCA9)
    for world in (2, 4, 8):
        for bad in ((), (100,)):
            doc, _ = _array_doc(rng, 6000, bad)
            a = np.frombuffer(doc, dtype=np.uint8)
            cuts = sharding.shard_cuts_at_lines(a, world, window=len(a) // (2 * world))
            short = rng.randrange(world)
            caps = [None] * world
            caps[short] = 64
            outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(world)], _stage1_body(caps))
            w = port.stage1(a)
            want = port.tokens(a, w.idx, w.n)
            for r, o in enumerate(outs):
                assert o["short_ranks"] == 1 << short and o["dirty_cuts"] == 0, (world, r)
                if bad:
                    assert o["rc"] == want[0] != 0 and o["first_error_index"] == want[6], (world, r)
                else:
                    assert o["rc"] == sj.CAPACITY and o["first_error_index"] == NONE64, (world, r)
                assert o["total_string_bytes"] == want[4]
            # the ranks that were not short wrote their part of the string buffer
            for r, o in enumerate(outs):
                if r != short:
                    assert o["sb"] == bytes(want[3][o["string_base"]: o["string_base"] + o["string_bytes"]]), (world, r)


def test_dirty_cut_is_refused(port):
    """a cut inside a string (shard_cuts, arbitrary bytes): UNEXPECTED_ERROR on every rank with the dirty ranks' bits,
    at once -- nobody waits for a round that does not come"""
    rng = random.Random(corpus.SEED ^ 0xD17)
    rows = [_row(rng, k) for k in range(2000)]
    big = b'{"k": "' + b"long string, no line feeds " * 20000 + b'"}'  # ~0.5 MB: the middle of the document, where every world cuts
    doc = b"[\n" + b",\n".join(rows[:1000] + [big] + rows[1000:]) + b"\n]"
    a = np.frombuffer(doc, dtype=np.uint8)
    for world in (2, 4, 8):
        cuts = sharding.shard_cuts(a, world)
        t0 = time.monotonic()
        outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(world)], _stage1_body())
        elapsed = time.monotonic() - t0
        dirty = sum(1 << r for r, o in enumerate(outs) if o["stage1_state_in"] != 0)
        assert dirty != 0
        for o in outs:
            assert o["rc"] == o["error"] == sj.UNEXPECTED_ERROR and o["dirty_cuts"] == dirty, (world, o["dirty_cuts"], dirty)
        assert elapsed < 15, elapsed


def test_whitespace_only_shard(port):
    doc = b'[1, "a",\n' + b" " * 70000 + b"\n" + b"\t" * 50000 + b'\n"b", 2.5e3, null]\n'
    a = np.frombuffer(doc, dtype=np.uint8)
    w = port.stage1(a)
    want = _whole(port, a, w.idx, w.n)
    for cuts in ([0, 9, 70010, len(doc)], [0, 20000, 40000, 60000, 90000, len(doc)]):
        outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(len(cuts) - 1)], _stage1_body())
        assert any(len(o["types"]) == 0 for o in outs)
        _check(outs, want, cuts)


def test_stream_and_comma_delimited_passes(port):
    """tokens over `kept` of an NDJSON stream pass (STREAMING_FINAL) and of a comma-delimited pass (COMMA_DELIMITED_FINAL)"""
    rows = [r for r in bytes(corpus.ndjson_rows(3 << 20)).split(b"\n") if r]
    cases = [(O.STREAMING_FINAL, b"\n".join(rows) + b"\n"), (O.COMMA_DELIMITED_FINAL, b",\n".join(rows) + b"\n")]
    L = sj.lib()
    for mode, doc in cases:
        a = np.frombuffer(doc, dtype=np.uint8)
        w = port.stage1(a, mode)
        assert w.err == 0
        want = _whole(port, a, w.idx, w.n)
        for world in (2, 4, 8):
            cuts = sharding.shard_cuts_at_lines(a, world, window=len(a) // (2 * world))

            def body(r, comm, p, d, stream):
                d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
                last = r == comm.world - 1
                if mode == O.STREAMING_FINAL:
                    rc, x = comm.scan_stream(d, d_idx, last, mode, stream)
                    st = x
                else:
                    rc, x = comm.scan_delimited(d, d_idx, last, mode, stream)
                    st = x.stream
                assert rc == 0, rc
                shard_len = int(st.total_bytes - st.bytes_before) if last else d.numel()
                return _tokens(comm, d[:shard_len], d_idx, int(st.kept), int(st.shard.state_in), stream)

            outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(world)], body)
            _check(outs, want, (mode, world))


def test_passes_of_other_kinds_in_flight(port):
    """tokens passes enqueued between stage-1 and minify passes on one comm, finished in order; finishing the oldest pass
    with the call of another kind leaves it in flight"""
    rng = random.Random(corpus.SEED ^ 0x1F1)
    doc, _ = _array_doc(rng, 8000, (4000,))
    a = np.frombuffer(doc, dtype=np.uint8)
    w = port.stage1(a)
    want = port.tokens(a, w.idx, w.n)
    _, want_min = port.minify(a)
    L = sj.lib()
    for world in (2, 4, 8):
        cuts = sharding.shard_cuts_at_lines(a, world, window=len(a) // (2 * world))

        def body(r, comm, p, d, stream):
            last = r == comm.world - 1
            d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
            d_idx2 = torch.empty_like(d_idx)
            dst = torch.empty(d.numel(), dtype=torch.uint8, device="cuda")
            rc, x = comm.scan(d, d_idx, last, stream)
            assert rc == 0
            n = int(x.count)
            assert comm.tokens_enqueue(d, d_idx, n, 0, None, stream) == 0
            assert comm.minify_enqueue(d, dst, stream) == 0
            assert comm.tokens_enqueue(d, d_idx, n, 0, None, stream) == 0
            assert comm.enqueue(d, d_idx2, last, stream) == 0
            assert comm.tokens_enqueue(d, d_idx, n, 0, None, stream) == 0
            res = [_fields(*comm.tokens_finish())]
            rc, _, t, _, _ = comm.tokens_finish()  # the oldest is the minify pass
            assert rc == sj.UNEXPECTED_ERROR and t is None and "another kind" in p.last_cuda_error()
            rc, xm = comm.minify_finish()
            assert rc == 0
            res.append(_fields(*comm.tokens_finish()))
            rc, x2 = comm.finish()
            assert rc == 0 and int(x2.count) == n
            res.append(_fields(*comm.tokens_finish()))
            torch.cuda.synchronize()
            return res, bytes(dst[: int(xm.count)].cpu().numpy())

        outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(world)], body)
        assert b"".join(o[1] for o in outs) == want_min
        for k in range(3):
            _check([o[0][k] for o in outs], want, (world, k))


def test_kind_mismatch_between_ranks(port):
    """rank 0 enqueues tokens where rank 1 enqueues minify: both fail, nothing hangs, and the comm works afterwards"""
    rng = random.Random(corpus.SEED ^ 0x2F2)
    doc, _ = _array_doc(rng, 3000)
    a = np.frombuffer(doc, dtype=np.uint8)
    cuts = sharding.shard_cuts_at_lines(a, 2)
    L = sj.lib()

    def body(r, comm, p, d, stream):
        d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        rc, x = comm.scan(d, d_idx, r == 1, stream)
        assert rc == 0
        dst = torch.empty(d.numel(), dtype=torch.uint8, device="cuda")
        if r == 0:
            rc1 = comm.tokens(d, d_idx, int(x.count), 0, None, stream)[0]
        else:
            rc1 = comm.minify(d, dst, stream)[0]
        err = p.last_cuda_error()
        f = _tokens(comm, d, d_idx, int(x.count), 0, stream)
        return rc1, err, f

    outs = _run_ranks([a[cuts[r]: cuts[r + 1]] for r in range(2)], body)
    assert all(o[0] == sj.UNEXPECTED_ERROR and "another kind" in o[1] for o in outs)
    w = port.stage1(a)
    _check([o[2] for o in outs], port.tokens(a, w.idx, w.n), "after the mismatch")


def test_one_rank_comm_matches_tokens_dev(port):
    rng = random.Random(corpus.SEED ^ 0x3F3)
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(4 << 20)
    assert rc == sj.SUCCESS
    comm = sharding.Comm(p, 0, 1)
    try:
        docs = _fuzz_docs(rng, 3) + [_array_doc(rng, 5000)[0], b"   \n  ", b'["' + b"x" * 5000 + b'", 1]']
        for doc in docs:
            a = np.frombuffer(doc, dtype=np.uint8)
            d = torch.from_numpy(a.copy()).cuda()
            d_idx = torch.empty(int(sj.lib().sjb200_index_words(len(a))), dtype=torch.int32, device="cuda")
            rc, x = comm.scan(d, d_idx, True)
            n = int(x.count)
            for cap in (None, 16):
                res, t1, p1, s1 = p.tokens_device(d, d_idx, n, cap)
                rc2, y, t2, p2, s2 = comm.tokens(d, d_idx, n, int(x.state_in), cap)
                torch.cuda.synchronize()
                assert rc2 == y.error == res.error and y.n_strings == res.n_strings and y.string_bytes == res.string_bytes, (doc[:40], cap)
                assert y.first_error_index == (NONE64 if res.first_error_index == 0xFFFFFFFF else res.first_error_index)
                assert y.short_ranks == (1 if res.string_bytes > (cap if cap is not None else s1.numel()) else 0)
                assert torch.equal(t1, t2) and torch.equal(p1, p2)
                if y.short_ranks == 0:
                    assert torch.equal(s1[: res.string_bytes], s2[: res.string_bytes])
    finally:
        comm.close()
        p.close()
