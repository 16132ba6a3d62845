"""Sharded stage-2 grammar (sjb200_document_errors_sharded*): a stream or one document cut into 1 / 2 / 4 / 8 shards after
line feeds, run through sharded stage 1 (plain, streaming-final, comma-delimited), the per-rank document tables, sharded
tokens and the sharded grammar; all ranks as threads of this process on one GPU (connect_local).  The results gathered
over the ranks must equal sjb200_document_errors_dev on the gathered arrays, and every rank must return the same finish
output.  Also: documents and errors at the cuts, depth limits at the cuts, ranks with 0, 1 and 2 structurals, passes of
other kinds in flight, kind / whole / max_depth mismatches, a bad table, CAPACITY with a fenced output, one-rank comms."""
import random

import numpy as np
import pytest
import torch

import grammar_oracle as G
import oracle_lib as O
import simdjson_b200 as sj
from simdjson_b200 import capi, corpus
from test_sharded_minify_utf8 import _run_ranks
from test_sharded_tokens import _array_doc

pytestmark = pytest.mark.gpu

NONE64 = (1 << 64) - 1
SAME = ("error", "first_error", "ndocs", "ndocs_in_error", "first_doc_in_error", "first_error_index")


def _lines(doc, world):
    """cuts right after line feeds, near equal shares (duplicates allowed: they make empty shards impossible, so skip)"""
    nl = [i + 1 for i, b in enumerate(doc) if b == 0x0A and i + 1 < len(doc)]
    cuts = [0]
    for k in range(1, world):
        want = len(doc) * k // world
        c = min(nl, key=lambda x: abs(x - want)) if nl else len(doc)
        cuts.append(max(c, cuts[-1]))
    cuts.append(len(doc))
    return cuts


def _body(mode, whole, max_depth=1024, tamper=None):
    """sharded stage 1 in `mode` (None: plain), the table (table mode), tokens, then the grammar pass"""
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
        rc, y, t, pay, _ = comm.tokens(d[:shard_len], d_idx, n, state_in, None, stream)
        assert y.dirty_cuts == 0 and y.short_ranks == 0, (rc, y.dirty_cuts)
        md, wh = max_depth, whole
        if tamper is not None:
            table, md, wh = tamper(r, table, md, wh)
        rc, res, errs, idxs = comm.document_errors(t, pay, n, wh, table, md, stream)
        torch.cuda.synchronize()
        f = {name: int(getattr(res, name)) for name, _ in capi.ShardedDocumentErrorsResult._fields_} if res is not None else {}
        f.update(rc=rc, last_error=p.last_cuda_error(), types=t.cpu().numpy().copy(), pay=pay.cpu().numpy().copy(), table=table, errs=errs, idxs=idxs, n=n)
        return f
    return body


def _unsharded(outs, whole, max_depth):
    types = np.concatenate([o["types"] for o in outs]).astype(np.uint8)
    pay = np.concatenate([o["pay"] for o in outs])
    base, starts = 0, []
    for o in outs:
        if not whole and o["table"] is not None and len(o["table"]):
            starts += [int(i) + base for i in np.asarray(o["table"])[:, 0]]
        base += o["n"]
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(1 << 16)
    assert rc == sj.SUCCESS
    try:
        d_type = torch.from_numpy(types).cuda()
        d_pay = torch.from_numpy(pay).cuda()
        d_docs = None
        if not whole and starts:
            d_docs = torch.from_numpy(np.array([[s, 0] for s in starts], dtype=np.uint32).view(np.int32).reshape(-1)).cuda()
        res, e, i = p.document_errors_device(d_type, d_pay, d_docs, len(starts) if d_docs is not None else None, max_depth)
        torch.cuda.synchronize()
        e, i = e.cpu().numpy(), i.cpu().numpy().view(np.uint32)
    finally:
        p.close()
    # the grammar oracle (sjo_document_errors) on the same gathered tokens: a check that shares no code with the kernels
    oe, oi = _gram().errors(types, pay, starts if not whole else None, max_depth)
    if whole or starts:
        assert np.array_equal(oe, e) and np.array_equal(oi, i), "the unsharded call differs from the grammar oracle"
    return res, e, i, len(starts)


_GRAM = []


def _gram():
    if not _GRAM:
        _GRAM.append(G.Grammar())
    return _GRAM[0]


def _check(outs, whole, max_depth, what):
    for r, o in enumerate(outs):
        assert o["rc"] == o["error"], (what, r, o["rc"])
        for k in SAME:
            assert o[k] == outs[0][k], (what, r, k, o[k], outs[0][k])
    tokens = docs = 0
    for r, o in enumerate(outs):
        assert (o["tokens_before"], o["docs_before"]) == (tokens, docs), (what, r)
        tokens += o["n"]
        docs += len(o["errs"]) if not whole else (1 if r == 0 else 0)
    res, e, i, nstarts = _unsharded(outs, whole, max_depth)
    if not whole and nstarts == 0:
        assert outs[0]["rc"] == 0 and outs[0]["ndocs"] == 0 and all(len(o["errs"]) == 0 for o in outs), what
        return e
    got_e = np.concatenate([o["errs"] for o in (outs[:1] if whole else outs)])
    got_i = np.concatenate([o["idxs"] for o in (outs[:1] if whole else outs)]).astype(np.uint64)
    want_i = np.where(i == 0xFFFFFFFF, np.uint64(NONE64), i.astype(np.uint64))
    assert len(got_e) == len(e) and np.array_equal(got_e, e), (what, list(zip(got_e[:8], e[:8])))
    assert np.array_equal(got_i, want_i), (what, [(k, got_i[k], want_i[k]) for k in np.nonzero(got_i != want_i)[0][:6]])
    o = outs[0]
    assert o["rc"] == 0 and o["ndocs"] == len(e), what
    assert o["ndocs_in_error"] == res.ndocs_in_error, (what, o["ndocs_in_error"], res.ndocs_in_error)
    fd = res.first_doc_in_error
    assert o["first_doc_in_error"] == (NONE64 if fd == 0xFFFFFFFF else fd), what
    if fd != 0xFFFFFFFF:
        assert (o["first_error"], o["first_error_index"]) == (int(e[fd]), int(want_i[fd])), what
    return e


def _run(doc, world, mode, whole, max_depth=1024, cuts=None, what=None):
    a = np.frombuffer(doc, dtype=np.uint8)
    cuts = cuts or _lines(doc, world)
    if any(cuts[k + 1] <= cuts[k] for k in range(len(cuts) - 1)):
        return None
    outs = _run_ranks([a[cuts[k]: cuts[k + 1]] for k in range(len(cuts) - 1)], _body(mode, whole, max_depth))
    return _check(outs, whole, max_depth, what or (world, mode, whole, max_depth, cuts))


def _ndjson(rng, nrows, bad):
    rows = [r for r in bytes(corpus.ndjson_rows(nrows * 300)).split(b"\n") if r][:nrows]
    for k in bad:
        if k < len(rows):
            rows[k] = rng.choice([rows[k][:-1], rows[k] + b"]", b"[" + rows[k], rows[k].replace(b":", b" ", 1), rows[k].replace(b",", b"", 1)])
    return rows


def test_ndjson_rows_with_corrupt_rows():
    rng = random.Random(corpus.SEED ^ 0x6A1)
    rows = _ndjson(rng, 3000, (0, 5, 777, 1500, 2998, 2999))
    for mode, sep in ((O.STREAMING_FINAL, b"\n"), (O.COMMA_DELIMITED_FINAL, b",\n")):
        doc = sep.join(rows) + b"\n"
        for world in (1, 2, 4, 8):
            e = _run(doc, world, mode, False)
            assert e is not None and (e != 0).sum() >= 4


def test_one_document_across_ranks():
    rng = random.Random(corpus.SEED ^ 0x6A2)
    good, _ = _array_doc(rng, 4000)
    bad, _ = _array_doc(rng, 4000, (10, 3999))
    docs = [good, bad, good[:-3] + b"\n", good.replace(b"},\n", b"}\n", 1), good.replace(b",\n", b"\n,", 2)]
    for doc in docs:
        for world in (2, 4, 8):
            _run(doc, world, None, True)
    for md in (1, 2, 3, 4):
        _run(good, 4, None, True, md)


def test_pretty_documents_across_cuts():
    """concatenated pretty-printed documents, cut after line feeds so that documents span ranks"""
    rng = random.Random(corpus.SEED ^ 0x6A3)
    docs = []
    for k in range(300):
        d = {"id": k, "a": [1, {"b": [2, 3, {}]}, []], "s": "x" * rng.randrange(5), "o": {"p": {"q": [None, True]}}}
        import json
        t = json.dumps(d, indent=rng.choice([1, 2])).encode()
        if k % 37 == 5:
            t = t.replace(b",", b"", 1)           # a missing comma
        if k % 41 == 7:
            t = t + b"\n]"                        # a stray closer
        if k % 43 == 9:
            t = t[:-2]                            # unclosed
        docs.append(t)
    stream = b"\n".join(docs) + b"\n"
    for world in (2, 4, 8):
        for shift in (0, 1, 2):
            cuts = _lines(stream, world)
            nl = [i + 1 for i, b in enumerate(stream) if b == 0x0A]
            cuts = [0] + [nl[min(len(nl) - 1, nl.index(c) + shift)] if c in nl else c for c in cuts[1:-1]] + [len(stream)]
            _run(stream, world, O.STREAMING_FINAL, False, cuts=cuts)


def _cut_after(doc, marks):
    """cuts after the line feeds that follow each mark"""
    cuts, at = [0], 0
    for m in marks:
        at = doc.index(m, at) + len(m)
        cuts.append(doc.index(b"\n", at) + 1 if doc[at - 1:at] != b"\n" else at)
    cuts.append(len(doc))
    return cuts


CUT_CASES = [
    # (stream, marks after whose line feed a cut falls, whole)
    (b'{"a": 1\n "b": 2}\n{"c": 3}\n', [b"1"], False),                       # a missing comma at a rank's first structural
    (b'[1, 2]\n]\n[3]\n', [b"2]"], False),                                   # a stray closer at a rank's start
    (b'{"key"\n: 1, "k2"\n:\n2}\n', [b'"key"', b'"k2"'], True),              # a key and its colon on two ranks
    (b'[[\n]]\n', [b"[["], True),                                            # an empty pair split by the cut
    (b'{"a": {\n}, "b": [\n]}\n', [b"{", b"["], True),
    (b'[1]\n[2]\n[3]\n', [b"[1]", b"[2]"], False),                           # documents that end exactly at cuts
    (b'[1]\n[2, [3\n', [b"[1]"], False),                                     # an unclosed document on the last rank
    (b'[\n1\n]\n', [b"[", b"1"], True),                                      # the root bracket's match on another rank; n = 1
    (b'[\n1,\n2\n]\n', [b"[", b"1,"], True),                                 # n = 2 between others
    (b'[\n\n\n1]\n', [b"[", b"\n"], True),                                   # a rank with n = 0
    (b'{"a":\n[1, 2]\n}\n', [b'"a":'], True),
    (b'1\n2\n3\n', [b"1", b"2"], False),
    (b'[1,\n]\n', [b"1,"], True),
]


def test_cut_cases():
    for doc, marks, whole in CUT_CASES:
        cuts = _cut_after(doc, marks)
        cuts = sorted(set(cuts))
        if any(cuts[k + 1] <= cuts[k] for k in range(len(cuts) - 1)):
            continue
        _run(doc, len(cuts) - 1, O.STREAMING_FINAL if not whole else None, whole, cuts=cuts, what=(doc, cuts))


@pytest.mark.parametrize("md", [1, 31, 32, 33, 1024, 4096])
def test_depth_limit_at_the_cut(md):
    """max_depth reached exactly at the cut, one below and one above, and empty pairs at the limit"""
    for depth in (md - 1, md, md + 1):
        if depth < 1:
            continue
        inner = b"[" * depth + b"\n" + b"]" * depth
        empty = b"[" * (depth - 1) + b"[\n]" + b"]" * (depth - 1)
        for doc, mark in ((inner + b"\n", b"[" * depth), (empty + b"\n", b"[" * depth), (b"[1]\n" + inner + b"\n[2]\n", b"[1]\n" + b"[" * depth)):
            cuts = _cut_after(doc, [mark])  # right after the opener at the limit (the empty pair's closer starts the next rank)
            _run(doc, 2, O.STREAMING_FINAL, False, md, cuts=sorted(set(cuts)), what=(md, depth, len(doc)))
            if doc.startswith(b"["):
                _run(doc, 2, None, True, md, cuts=sorted(set(cuts)), what=(md, depth, "whole"))


def test_passes_of_other_kinds_in_flight():
    rng = random.Random(corpus.SEED ^ 0x6A4)
    rows = _ndjson(rng, 800, (3, 400))
    doc = b"\n".join(rows) + b"\n"
    a = np.frombuffer(doc, dtype=np.uint8)
    L = sj.lib()
    for world in (2, 4):
        cuts = _lines(doc, world)

        def body(r, comm, p, d, stream):
            last = r == comm.world - 1
            d_idx = torch.empty(int(L.sjb200_index_words(d.numel())), dtype=torch.int32, device="cuda")
            d_idx2 = torch.empty_like(d_idx)
            rc, x = comm.scan_stream(d, d_idx, last, O.STREAMING_FINAL, stream)
            assert rc == 0
            n = int(x.kept)
            table = comm.document_table(d, d_idx, x, stream)
            shard_len = int(x.total_bytes - x.bytes_before) if last else d.numel()
            _, _, t, pay, _ = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)
            assert comm.document_errors_enqueue(t, pay, n, False, table, None, stream) == 0
            assert comm.tokens_enqueue(d[:shard_len], d_idx, n, 0, None, stream) == 0
            assert comm.enqueue(d, d_idx2, last, stream) == 0
            assert comm.document_errors_enqueue(t, pay, n, False, table, None, stream) == 0
            res = [comm.document_errors_finish()]
            rc = comm.document_errors_finish()[0]  # the oldest is the tokens pass
            assert rc == sj.UNEXPECTED_ERROR and "another kind" in p.last_cuda_error()
            assert comm.tokens_finish()[0] not in (sj.UNEXPECTED_ERROR, sj.CAPACITY)
            assert comm.finish()[0] == 0
            res.append(comm.document_errors_finish())
            torch.cuda.synchronize()
            return [dict({name: int(getattr(y, name)) for name, _ in capi.ShardedDocumentErrorsResult._fields_}, rc=rc2, errs=e, idxs=i, n=n, table=table,
                         types=t.cpu().numpy().copy(), pay=pay.cpu().numpy().copy()) for rc2, y, e, i in res]

        outs = _run_ranks([a[cuts[k]: cuts[k + 1]] for k in range(world)], body)
        for k in range(2):
            _check([o[k] for o in outs], False, 1024, (world, k))


def _rows_doc():
    rng = random.Random(corpus.SEED ^ 0x6A5)
    rows = _ndjson(rng, 400, (7,))
    return b"\n".join(rows) + b"\n"


def test_mismatches_and_bad_table():
    doc = _rows_doc()
    a = np.frombuffer(doc, dtype=np.uint8)
    cuts = _lines(doc, 4)
    shards = [a[cuts[k]: cuts[k + 1]] for k in range(4)]
    # whole / max_depth disagree: UNEXPECTED_ERROR on every rank, at once, with no results
    for tamper in (lambda r, t, md, wh: (t, 512 if r == 2 else md, wh), lambda r, t, md, wh: (t, md, r == 1)):
        outs = _run_ranks(shards, _body(O.STREAMING_FINAL, False, 1024, tamper))
        assert all(o["rc"] == sj.UNEXPECTED_ERROR and "disagree" in o["last_error"] and len(o["errs"]) == 0 for o in outs)
    # a bad table on one rank: UNEXPECTED_ERROR everywhere, every result {UNEXPECTED_ERROR, none}
    def bad(r, t, md, wh):
        if r == 1 and len(t) >= 2:
            t = t.copy()
            t[1, 0] = t[0, 0]
        return t, md, wh
    outs = _run_ranks(shards, _body(O.STREAMING_FINAL, False, 1024, bad))
    for o in outs:
        assert o["rc"] == sj.UNEXPECTED_ERROR and o["first_doc_in_error"] == 0 and o["ndocs_in_error"] == o["ndocs"] > 0
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
        _, _, t, pay, _ = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)
        d_docs = torch.from_numpy(np.ascontiguousarray(table.astype(np.uint32)).view(np.int32).reshape(-1)).cuda()
        fence = torch.full((len(table) * 2 + 8,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
        res = capi.ShardedDocumentErrorsResult()
        rc = L.sjb200_document_errors_sharded(comm._h, t.data_ptr(), pay.data_ptr(), n, 0, d_docs.data_ptr(), len(table), 0 if r == 0 else 1024,
                                              fence[4:].data_ptr(), res, stream.cuda_stream)
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
        _, _, t, pay, _ = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)
        if r == 0:
            rc1 = comm.document_errors(t, pay, n, False, table, None, stream)[0]
        else:
            rc1 = comm.tokens(d[:shard_len], d_idx, n, 0, None, stream)[0]
        err = p.last_cuda_error()
        rc2 = comm.document_errors(t, pay, n, False, table, None, stream)[0]
        return rc1, err, rc2

    outs = _run_ranks([a[cuts[k]: cuts[k + 1]] for k in range(2)], body)
    assert all(o[0] == sj.UNEXPECTED_ERROR and "another kind" in o[1] for o in outs), outs
    assert all(o[2] == 0 for o in outs), outs


def test_one_rank_comm_matches_document_errors_dev():
    rng = random.Random(corpus.SEED ^ 0x6A6)
    doc = b"\n".join(_ndjson(rng, 500, (1, 250))) + b"\n"
    _run(doc, 1, O.STREAMING_FINAL, False)
    good, _ = _array_doc(rng, 500)
    _run(good, 1, None, True)
    _run(b"  \n", 1, None, True)
