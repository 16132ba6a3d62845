"""Sharded JSON Pointer lookup (sjb200_at_pointer_sharded*): a stream or one document cut into 1 to 8 shards after line
feeds, run through sharded stage 1 (plain, streaming-final, comma-delimited), the per-rank document tables, sharded
tokens and the sharded pointer pass; all ranks as threads of this process on one GPU (connect_local).  The results
gathered over the ranks must equal sjb200_at_pointer_dev on the gathered arrays (and, on a sample of documents, the
pointer oracle), and every rank must return the same finish output.  Also: walks that cross cuts in every way the
continuation record covers, token errors on later ranks, passes of other kinds in flight, kind / whole / pointer-set
mismatches, a bad table, CAPACITY with a fenced output, one-rank comms, and the drop-by-verdict rule."""
import json
import random

import numpy as np
import pytest
import torch

import oracle_lib as O
import pointer_cases as PC
import pointer_oracle as PO
import simdjson_b200 as sj
from simdjson_b200 import capi, corpus
from test_sharded_document_errors import _cut_after, _lines
from test_pointer_shards_emul import nested_ok
from test_sharded_minify_utf8 import _run_ranks

pytestmark = pytest.mark.gpu

NONE64 = (1 << 64) - 1
SAME = ("error", "rounds", "ndocs")
_PO = []


def _oracle():
    if not _PO:
        _PO.append(PO.Pointers())
    return _PO[0]


def _body(mode, whole, pointers, tamper=None, verdict=False):
    """sharded stage 1 in `mode` (None: plain), the table (table mode), tokens, then the pointer pass"""
    L = sj.lib()

    def body(r, comm, p, d, stream):
        last = r == comm.world - 1
        d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        table = None
        if mode is None:
            rc, x = comm.scan(d, d_idx, last, stream)
            n, state_in, shard_len = int(x.count), int(x.state_in), d.numel()
        else:
            if mode == O.STREAMING_FINAL:
                rc, x = comm.scan_stream(d, d_idx, last, mode, stream)
                st = x
            else:
                rc, x = comm.scan_delimited(d, d_idx, last, mode, stream)
                st = x.stream
            n, state_in = int(st.kept), int(st.shard.state_in)
            shard_len = int(st.total_bytes - st.bytes_before) if last else d.numel()
            if not whole:
                table = comm.document_table(d, d_idx, st, stream)
        assert rc == 0, rc
        rc, y, t, pay, sb = comm.tokens(d[:shard_len], d_idx, n, state_in, None, stream)
        assert y.dirty_cuts == 0 and y.short_ranks == 0, (rc, y.dirty_cuts)
        ptrs, wh = pointers, whole
        if tamper is not None:
            table, ptrs, wh = tamper(r, table, ptrs, wh)
        sbytes = int(y.string_bytes)
        rc, res, errs, idxs = comm.at_pointer(ptrs, t, pay, n, sb, sbytes, wh, table, stream)
        torch.cuda.synchronize()
        f = {name: int(getattr(res, name)) for name, _ in capi.ShardedPointerSummary._fields_} if res is not None else {}
        f.update(rc=rc, last_error=p.last_cuda_error(), types=t.cpu().numpy().copy(), pay=pay.cpu().numpy().view(np.uint64).copy(),
                 strbuf=sb[:sbytes].cpu().numpy().copy(), string_base=int(y.string_base), table=table, errs=errs, idxs=idxs, n=n, grammar=None)
        if verdict:
            f["grammar"] = comm.document_errors(t, pay, n, wh, table, None, stream)[2]
        return f
    return body


def _gather(outs, whole):
    types = np.concatenate([o["types"][: o["n"]] for o in outs]).astype(np.uint8)
    pays = []
    for o in outs:
        pl = o["pay"][: o["n"]].copy()
        pl[o["types"][: o["n"]] == ord('"')] += np.uint64(o["string_base"])
        pays.append(pl)
    pay = np.concatenate(pays) if pays else np.zeros(0, np.uint64)
    strbuf = np.concatenate([o["strbuf"] for o in outs]).astype(np.uint8)
    base, starts = 0, []
    for o in outs:
        if not whole and o["table"] is not None and len(o["table"]):
            starts += [int(i) + base for i in np.asarray(o["table"])[:, 0]]
        base += o["n"]
    return types, pay, strbuf, starts


def _unsharded(types, pay, strbuf, starts, whole, pointers):
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(1 << 16)
    assert rc == sj.SUCCESS
    try:
        d_type = torch.from_numpy(types if len(types) else np.zeros(1, np.uint8)).cuda()[: len(types)]
        d_pay = torch.from_numpy((pay if len(pay) else np.zeros(1, np.uint64)).view(np.int64)).cuda()[: len(types)]
        d_sb = torch.from_numpy(strbuf if len(strbuf) else np.zeros(1, np.uint8)).cuda()
        d_docs = None
        if not whole and starts:
            d_docs = torch.from_numpy(np.array([[s, 0] for s in starts], dtype=np.uint32).view(np.int32).reshape(-1)).cuda()
        e, i = p.at_pointer_device(pointers, d_type, d_pay, d_sb, len(strbuf), d_docs, len(starts) if d_docs is not None else None)
        torch.cuda.synchronize()
        return e.cpu().numpy(), i.cpu().numpy().view(np.uint32)
    finally:
        p.close()


def _check(outs, whole, pointers, what, oracle_docs=6):
    for r, o in enumerate(outs):
        assert o["rc"] == o["error"], (what, r, o["rc"], o["last_error"])
        for k in SAME:
            assert o[k] == outs[0][k], (what, r, k, o[k], outs[0][k])
    tokens = docs = 0
    for r, o in enumerate(outs):
        assert (o["tokens_before"], o["docs_before"]) == (tokens, docs), (what, r)
        tokens += o["n"]
        docs += o["errs"].shape[1] if not whole else (1 if r == 0 else 0)
    types, pay, strbuf, starts = _gather(outs, whole)
    if not whole and not starts:
        assert all(o["rc"] == 0 and o["ndocs"] == 0 and o["errs"].size == 0 for o in outs), what
        return None
    e, i = _unsharded(types, pay, strbuf, starts, whole, pointers)
    got_e = np.concatenate([o["errs"] for o in (outs[:1] if whole else outs)], axis=1)
    got_i = np.concatenate([o["idxs"] for o in (outs[:1] if whole else outs)], axis=1).astype(np.uint64)
    want_i = np.where(i == 0xFFFFFFFF, np.uint64(NONE64), i.astype(np.uint64))
    assert got_e.shape == e.shape and np.array_equal(got_e, e), (what, [(p, d, got_e[p, d], e[p, d]) for p, d in zip(*np.nonzero(got_e != e))][:6])
    assert np.array_equal(got_i, want_i), (what, [(p, d, got_i[p, d], want_i[p, d]) for p, d in zip(*np.nonzero(got_i != want_i))][:6])
    assert outs[0]["rc"] == 0 and outs[0]["ndocs"] == e.shape[1], what
    # the pointer oracle (sjo_at_pointer) on the gathered tokens, for the first and last documents and those at the cuts
    D = e.shape[1]
    cut_docs = set()
    for o in outs:
        if not whole and starts:
            cut_docs.add(max(0, int(np.searchsorted(starts, o["tokens_before"], side="right")) - 1))
    sample = sorted({d for d in list(range(min(oracle_docs, D))) + list(range(max(0, D - oracle_docs), D)) + list(cut_docs) if 0 <= d < D})
    for d in sample:
        s = 0 if whole else starts[d]
        end = len(types) if whole or d + 1 >= len(starts) else starts[d + 1]
        if not nested_ok(types, s, end) and 0 not in types[s:end]:
            continue  # the walk's documented deviation: the gathered call above is the reference
        for p, ptr in enumerate(pointers):
            oe, oi = _oracle().at_pointer(types, pay, strbuf, ptr, s, end)
            assert (oe, oi) == (int(e[p, d]), int(i[p, d])), (what, d, ptr, (oe, oi), (int(e[p, d]), int(i[p, d])))
    return got_e, got_i, outs


def _run(doc, world, mode, whole, pointers, cuts=None, what=None, tamper=None, verdict=False):
    a = np.frombuffer(doc, dtype=np.uint8)
    cuts = cuts or _lines(doc, world)
    if any(cuts[k + 1] <= cuts[k] for k in range(len(cuts) - 1)):
        return None
    outs = _run_ranks([a[cuts[k]: cuts[k + 1]] for k in range(len(cuts) - 1)], _body(mode, whole, pointers, tamper, verdict))
    return _check(outs, whole, pointers, what or (world, mode, whole, cuts))


TWITTER_POINTERS = ["/id", "/user/screen_name", "/entities/hashtags/0/text", "/retweet_count", "/nope", "/user/0", "", "x"]


def test_twitter_rows():
    rows = PC.twitter_rows()
    for mode, sep in ((O.STREAMING_FINAL, b"\n"), (O.COMMA_DELIMITED_FINAL, b",\n")):
        doc = sep.join(rows * 3) + b"\n"
        for world in (1, 2, 3, 4, 8):
            r = _run(doc, world, mode, False, TWITTER_POINTERS)
            assert r is not None
            assert all(o["rounds"] == 0 and o["walks_forwarded"] == 0 for o in r[2])  # rows cut after line feeds: nothing crosses


def _pretty_stream(rng, count):
    docs = []
    for k in range(count):
        d = {"id": k, "a": [1, {"b": [2, 3, {}]}, list(range(rng.randrange(40)))], "s": "x" * rng.randrange(5), "o": {"p": {"q": [None, True]}}}
        t = json.dumps(d, indent=rng.choice([1, 2])).encode()
        if k % 2 == 0:
            t = t.replace(b'"id"', b'"s": "first",\n"id"', 1)  # a duplicate key: the first match wins
        if k % 37 == 5:
            t = t.replace(b",", b"", 1)           # a missing comma
        if k % 41 == 7:
            t = t + b"\n]"                        # a stray closer
        if k % 43 == 9:
            t = t[:-2]                            # unclosed
        if k % 47 == 11:
            t = t.replace(b"true", b"tru", 1)     # a token in error at the end of the document
        docs.append(t)
    return b"\n".join(docs) + b"\n"


PRETTY_POINTERS = ["/a/1/b/2", "/a/2/17", "/a/2/39", "/a/3", "/o/p/q/1", "/o/p/q/2", "/o/p/x", "/s", "/id", "/a/1/b/-", "/o/p/q/0/z", "/a/x", "/o/~2"]


def test_pretty_documents_across_cuts():
    """concatenated pretty-printed documents cut after every few line feeds: documents, containers and arrays span ranks"""
    rng = random.Random(corpus.SEED ^ 0x7B1)
    stream = _pretty_stream(rng, 200)
    nl = [i + 1 for i, b in enumerate(stream) if b == 0x0A]
    forwarded = 0
    for world in (2, 3, 4, 8):
        for shift in (0, 1, 2, 5):
            cuts = _lines(stream, world)
            cuts = [0] + [nl[min(len(nl) - 1, nl.index(c) + shift)] if c in nl else c for c in cuts[1:-1]] + [len(stream)]
            r = _run(stream, world, O.STREAMING_FINAL, False, PRETTY_POINTERS, cuts=sorted(set(cuts)))
            if r is not None:
                forwarded += sum(o["walks_forwarded"] for o in r[2])
    assert forwarded > 0


def _spread(doc):
    """the document with a line feed after every structural character and scalar, so that a cut after a line feed can
    fall between any two structurals"""
    out, in_str, esc = bytearray(), False, False
    for b in doc:
        out.append(b)
        if in_str:
            if esc:
                esc = False
            elif b == 0x5C:
                esc = True
            elif b == 0x22:
                in_str = False
                out += b"\n"
            continue
        if b == 0x22:
            in_str = True
        elif b in b"{}[],:":
            out += b"\n"
    return bytes(out)


CUT_DOCS = [
    # (document, pointers, table)
    (b'{"key": {"x": [10, 20, 30]}, "b": 1}', ["/key/x/2", "/key/x/3", "/key/y", "/b", "/key/x/0/z", "/b/0", "/key/x/1/q/r", "/-"], False),
    (b'{"a": 1, "a": 2, "c": {"a": 3}}', ["/a", "/c/a", "/c/b", "/d"], False),
    (b'[[1, [2, [3, [4]]]], {"k": [[], {}]}, "s", 5]', ["/0/1/1/1/0", "/1/k/0", "/1/k/1/x", "/3", "/4", "/2/0", "/0/1/1/1/1"], False),
    (b'{"a": {}}\n{"a": []}\n{"a": [1, 2]}\n[{"a": 1}]\n"x"\n{"a": {"b": 1}}', ["/a", "/a/0", "/a/1", "/a/b", "/0/a", ""], True),
    (b'{"a": [1, tru, 3], "b": 2}\n{"b": [1, 2, 3]}', ["/b", "/a/0", "/b/2"], True),
    (b'{"a": [1, [2, 3}, "b": 2}\n{"b": {"c": ]]}', ["/b", "/a/1/1", "/b/c", "/a/1/5"], True),  # nesting errors across cuts
]


def test_cut_cases():
    """every placement of one and two cuts between the structurals of small documents: a key as a rank's last
    structural with its ':' on the next rank, a ':' last with the value next, containers opening at the cut, arrays
    counted across cuts, duplicate keys on two ranks, errors decided on a later rank, ranks of 0, 1 and 2 structurals"""
    for doc, pointers, table in CUT_DOCS:
        d = _spread(doc) + b"\n"
        nl = [i + 1 for i, b in enumerate(d) if b == 0x0A and i + 1 < len(d)]
        positions = nl if len(nl) <= 24 else nl[:: max(1, len(nl) // 24)]
        for whole in ((False,) if table else (False, True)):
            mode = O.STREAMING_FINAL if not whole else None
            for c in positions:
                _run(d, 2, mode, whole, pointers, cuts=[0, c, len(d)], what=(doc, whole, c))
            for j in range(0, len(positions) - 2, 3):
                a, b, c = positions[j], positions[j + 1], positions[j + 2]
                for world_cuts in ([0, a, b, len(d)], [0, a, b, c, len(d)]):  # ranks of 1 and 2 structurals between cuts
                    _run(d, len(world_cuts) - 1, mode, whole, pointers, cuts=sorted(set(world_cuts)), what=(doc, whole, world_cuts))



def test_whole_mode_targets_on_every_rank():
    """one array across 2, 3, 4 and 8 ranks: the first, middle and last root element, deep paths, errors past the end"""
    rng = random.Random(corpus.SEED ^ 0x7B2)
    elems = [{"i": i, "v": [i, str(i), {"d": [[i]]}]} if i % 3 else [i, [i, [i]]] for i in range(6000)]
    doc = b"[\n" + b",\n".join(json.dumps(e).encode() for e in elems) + b"\n]\n"
    pointers = ["/0", "/1/v/2/d/0/0", "/3000", "/2999/v/1", "/5999", "/5998/v/2/d/0", "/5999/1/1/0", "/6000", "/-", "/1/x", "/2/1/0/0", ""]
    for world in (2, 3, 4, 8):
        r = _run(doc, world, None, True, pointers)
        assert r is not None and r[2][0]["rounds"] == world - 1


def test_token_error_on_a_later_rank_wins():
    """a token in error in a later rank's leading segment beats a walk that would finish on the owner"""
    doc = b'{"a": 1, "b": [\n1, 2, 3,\n4, tru, 6]}\n{"a": 2}\n'
    cuts = _cut_after(doc, [b"[\n1, 2, 3,\n"])
    for mode in (O.STREAMING_FINAL,):
        r = _run(doc, 2, mode, False, ["/a", "/b/0", "/q", "x", ""], cuts=cuts)
        assert r is not None and (r[0][:, 0] != 0).all() and len(set(r[1][:, 0].tolist())) == 1 and r[1][0, 0] != NONE64


def test_pointer_passes_in_flight_with_other_kinds():
    rows = PC.twitter_rows()[:120]
    doc = b"\n".join(rows) + b"\n"
    a = np.frombuffer(doc, dtype=np.uint8)
    L = sj.lib()
    for world in (2, 4):
        cuts = _lines(doc, world)

        def body(r, comm, p, d, stream):
            last = r == comm.world - 1
            d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
            rc, x = comm.scan_stream(d, d_idx, last, O.STREAMING_FINAL, stream)
            assert rc == 0
            n = int(x.kept)
            table = comm.document_table(d, d_idx, x, stream)
            shard_len = int(x.total_bytes - x.bytes_before) if last else d.numel()
            _, y, t, pay, sb = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)
            sbytes = int(y.string_bytes)
            assert comm.at_pointer_enqueue(TWITTER_POINTERS, t, pay, n, sb, sbytes, False, table, stream) == 0
            assert comm.document_errors_enqueue(t, pay, n, False, table, None, stream) == 0
            assert comm.tokens_enqueue(d[:shard_len], d_idx, n, 0, None, stream) == 0
            assert comm.at_pointer_enqueue(TWITTER_POINTERS[::-1], t, pay, n, sb, sbytes, False, table, stream) == 0
            res = [comm.at_pointer_finish()]
            rc = comm.at_pointer_finish()[0]  # the oldest is the grammar pass
            assert rc == sj.UNEXPECTED_ERROR and "another kind" in p.last_cuda_error()
            assert comm.document_errors_finish()[0] == 0
            assert comm.tokens_finish()[0] == 0
            res.append(comm.at_pointer_finish())
            torch.cuda.synchronize()
            base = dict(types=t.cpu().numpy().copy(), pay=pay.cpu().numpy().view(np.uint64).copy(), strbuf=sb[:sbytes].cpu().numpy().copy(),
                        string_base=int(y.string_base), table=table, n=n, last_error="")
            return [dict(base, **{name: int(getattr(s, name)) for name, _ in capi.ShardedPointerSummary._fields_}, rc=rc2, errs=e, idxs=i)
                    for rc2, s, e, i in res]

        outs = _run_ranks([a[cuts[k]: cuts[k + 1]] for k in range(world)], body)
        _check([o[0] for o in outs], False, TWITTER_POINTERS, (world, 0))
        _check([o[1] for o in outs], False, TWITTER_POINTERS[::-1], (world, 1))


def _rows_doc():
    return b"\n".join(PC.twitter_rows()[:60]) + b"\n"


def test_mismatches_and_bad_table():
    doc = _rows_doc()
    a = np.frombuffer(doc, dtype=np.uint8)
    cuts = _lines(doc, 4)
    shards = [a[cuts[k]: cuts[k + 1]] for k in range(4)]
    for tamper in (lambda r, t, ps, wh: (t, ps[:-1] if r == 2 else ps, wh), lambda r, t, ps, wh: (t, ["/x"] + ps[1:] if r == 3 else ps, wh),
                   lambda r, t, ps, wh: (t, ps, r == 1)):
        outs = _run_ranks(shards, _body(O.STREAMING_FINAL, False, TWITTER_POINTERS, tamper))
        assert all(o["rc"] == sj.UNEXPECTED_ERROR and "disagree" in o["last_error"] and o["errs"].size == 0 for o in outs), [o["last_error"] for o in outs]

    def bad(r, t, ps, wh):
        if r == 1 and len(t) >= 2:
            t = t.copy()
            t[1, 0] = t[0, 0]
        return t, ps, wh
    outs = _run_ranks(shards, _body(O.STREAMING_FINAL, False, TWITTER_POINTERS, bad))
    for o in outs:
        assert o["rc"] == sj.UNEXPECTED_ERROR and o["ndocs"] > 0, o["last_error"]
        assert (o["errs"] == sj.UNEXPECTED_ERROR).all() and (o["idxs"] == np.uint64(NONE64)).all()


def test_capacity_with_fenced_output():
    doc = _rows_doc()
    a = np.frombuffer(doc, dtype=np.uint8)
    cuts = _lines(doc, 2)
    L = sj.lib()

    def body(r, comm, p, d, stream):
        last = r == 1
        d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        rc, x = comm.scan_stream(d, d_idx, last, O.STREAMING_FINAL, stream)
        n = int(x.kept)
        table = comm.document_table(d, d_idx, x, stream)
        shard_len = int(x.total_bytes - x.bytes_before) if last else d.numel()
        _, y, t, pay, sb = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)
        d_docs = torch.from_numpy(np.ascontiguousarray(table.astype(np.uint32)).view(np.int32).reshape(-1)).cuda()
        P = 1025 if r == 0 else 1024  # one rank over SJB200_POINTER_SHARDED_MAX_POINTERS
        enc = [b"/id"] * P
        import ctypes as C
        bufs = [C.create_string_buffer(e, len(e)) for e in enc]
        ptrs = (C.c_void_p * P)(*[C.addressof(b) for b in bufs])
        lens = (C.c_size_t * P)(*[len(e) for e in enc])
        fence = torch.full((P * len(table) * 2 + 8,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
        res = capi.ShardedPointerSummary()
        rc = L.sjb200_at_pointer_sharded(comm._h, t.data_ptr(), pay.data_ptr(), n, sb.data_ptr(), int(y.string_bytes), 0, d_docs.data_ptr(), len(table),
                                         ptrs, lens, P, fence[4:].data_ptr(), res, stream.cuda_stream)
        torch.cuda.synchronize()
        return rc, bool((fence == 0x5A5A5A5A5A5A5A5A).all())

    outs = _run_ranks([a[cuts[k]: cuts[k + 1]] for k in range(2)], body)
    assert all(o == (sj.CAPACITY, True) for o in outs), outs


def test_kind_mismatch_between_ranks():
    doc = _rows_doc()
    a = np.frombuffer(doc, dtype=np.uint8)
    cuts = _lines(doc, 2)
    L = sj.lib()

    def body(r, comm, p, d, stream):
        last = r == 1
        d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
        rc, x = comm.scan_stream(d, d_idx, last, O.STREAMING_FINAL, stream)
        n = int(x.kept)
        table = comm.document_table(d, d_idx, x, stream)
        shard_len = int(x.total_bytes - x.bytes_before) if last else d.numel()
        _, y, t, pay, sb = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)
        if r == 0:
            rc1 = comm.at_pointer(TWITTER_POINTERS, t, pay, n, sb, int(y.string_bytes), False, table, stream)[0]
        else:
            rc1 = comm.document_errors(t, pay, n, False, table, None, stream)[0]
        err = p.last_cuda_error()
        rc2 = comm.at_pointer(TWITTER_POINTERS, t, pay, n, sb, int(y.string_bytes), False, table, stream)[0]
        return rc1, err, rc2

    outs = _run_ranks([a[cuts[k]: cuts[k + 1]] for k in range(2)], body)
    assert all(o[0] == sj.UNEXPECTED_ERROR and "another kind" in o[1] for o in outs), outs
    assert all(o[2] == 0 for o in outs), outs


def test_one_rank_comm_matches_at_pointer_dev():
    rng = random.Random(corpus.SEED ^ 0x7B3)
    _run(_pretty_stream(rng, 50), 1, O.STREAMING_FINAL, False, PRETTY_POINTERS)
    _run(b"[\n" + b",\n".join(json.dumps({"i": i}).encode() for i in range(500)) + b"\n]\n", 1, None, True, ["/0/i", "/499/i", "/500"])


def test_drop_documents_whose_verdict_is_not_success():
    """the results of documents whose sjb200_document_errors_sharded verdict is SUCCESS equal the oracle on each of them
    parsed alone"""
    rng = random.Random(corpus.SEED ^ 0x7B4)
    stream = _pretty_stream(rng, 120)
    for world in (2, 4):
        got_e, got_i, outs = _run(stream, world, O.STREAMING_FINAL, False, PRETTY_POINTERS, verdict=True)
        verdict = np.concatenate([o["grammar"] for o in outs])
        types, pay, strbuf, starts = _gather(outs, False)
        good = np.nonzero(verdict == 0)[0]
        assert 0 < len(good) < len(verdict)
        for d in good[:: max(1, len(good) // 25)]:
            end = starts[d + 1] if d + 1 < len(starts) else len(types)
            assert nested_ok(types, starts[d], end)
            for p, ptr in enumerate(PRETTY_POINTERS):
                oe, oi = _oracle().at_pointer(types, pay, strbuf, ptr, starts[d], end)
                assert (got_e[p, d], got_i[p, d]) == (oe, NONE64 if oi == 0xFFFFFFFF else oi), (d, ptr)
