"""CPU check of the sharded stage-2-lite's key fact (sjb200_tokens_sharded*): at a clean cut -- scanner state 0 entering
the shard -- the token functions run on the shard alone (tests/tokens_emul.cpp, the kernels' decomposition on the host)
give exactly the whole document's tokens, rebased: '"' payloads by the string bytes of the earlier shards, 'd' payloads
by the shard's offset, the first error by the tokens of the earlier shards.  And at a cut with state != 0 they do not,
which is why the sharded call refuses such cuts.  The GPU run of the sharded call is tests/test_sharded_tokens.py."""
import ctypes as C
import random

import numpy as np

import oracle_lib as O
import token_fuzz as TF
from simdjson_b200 import corpus
from test_tokens_emul import emu, run_emu  # noqa: F401  (the fixture that builds tests/tokens_emul.cpp)

WS = b" \t\r\n"


def _state(port, buf):
    """the oracle's scanner state after buf (bit0 escape, bit1 in string, bit2 previous byte a non-quote scalar)"""
    L = port.L
    L.sjo_scan_shard.restype = C.c_uint64
    L.sjo_scan_shard.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    a = np.frombuffer(bytes(buf), dtype=np.uint8)
    so = C.c_uint32(0)
    L.sjo_scan_shard(a.ctypes.data if len(a) else None, len(a), 0, None, C.byref(so))
    return int(so.value)


def sharded(L, doc, idx, n, cuts):
    """every shard through the emulation, outputs rebased and concatenated, the first error folded as finish() does"""
    idx = np.asarray(idx[:n], dtype=np.int64)
    types, pays, sbuf = [], [], []
    err, first, tokens_before, string_base, nstr = 0, 0xFFFFFFFF, 0, 0, 0
    for r in range(len(cuts) - 1):
        lo, hi = cuts[r], cuts[r + 1]
        sel = idx[(idx >= lo) & (idx < hi)] - lo
        e, t, p, sb, sl, ns, fe = run_emu(L, doc[lo:hi], sel.astype(np.uint32), len(sel))
        p = p.copy()
        p[t == ord('"')] += np.uint64(string_base)
        p[t == ord("d")] += np.uint64(lo)
        if err == 0 and e not in (0, 1):
            err, first = e, tokens_before + fe
        types.append(bytes(t)); pays.append(p); sbuf.append(bytes(sb))
        tokens_before += len(sel); string_base += sl; nstr += ns
    return err, b"".join(types), np.concatenate(pays) if pays else np.zeros(0, np.uint64), b"".join(sbuf), string_base, nstr, first


def whole(port, doc, idx, n):
    e, t, p, sb, sl, ns, fe = port.tokens(doc, idx, n)
    return e, bytes(t), p, bytes(sb), sl, ns, fe


def same(a, b):
    return a[0] == b[0] and a[1] == b[1] and np.array_equal(a[2], b[2]) and a[3] == b[3] and a[4:] == b[4:]


def clean_cuts(port, doc, rng, nshards, kind):
    """nshards - 1 cuts of the given kind, each checked clean with the oracle: after a line feed, a closing quote, an
    operator, or inside a whitespace run"""
    def fits(p):
        prev = doc[p - 1]
        if kind == "lf":
            return prev == 0x0A
        if kind == "quote":
            return prev == 0x22
        if kind == "operator":
            return prev in b",:[]{}"
        return prev in WS and doc[p] in WS  # inside a whitespace run
    cuts = [0]
    for k in range(1, nshards):
        p = max(cuts[-1] + 1, len(doc) * k // nshards + rng.randrange(-len(doc) // (4 * nshards) - 1, len(doc) // (4 * nshards) + 1))
        while p < len(doc) and not (fits(p) and _state(port, doc[:p]) == 0):
            p += 1
        if p >= len(doc):
            break
        cuts.append(p)
    cuts.append(len(doc))
    return cuts


def _fuzz_docs(rng, count):
    """documents of adversarial tokens -- every scalar kind and string body the fuzzers make, errors included -- laid out
    over several lines so that errors land in every shard"""
    docs = []
    for _ in range(count):
        parts = []
        for _ in range(rng.randrange(200, 1500)):
            if rng.random() < 0.5:
                body, _bad = TF.string_body(rng)
                parts.append(b'"' + body + b'"')
            else:
                tok = TF.scalar_token(rng)
                if b'"' in tok or b"\\" in tok:
                    continue
                parts.append(tok)
        docs.append(b"[" + b"".join(p + rng.choice([b",", b" ,\n ", b", ", b",\n", b" :  "]) for p in parts) + b"0]")
    return docs


def test_clean_cuts_give_the_whole_documents_tokens(emu):  # noqa: F811
    port = O.Port()
    rng = random.Random(corpus.SEED ^ 0x70C5)
    docs = _fuzz_docs(rng, 12)
    docs += [bytes(corpus.random_json(rng.randrange(20000, 300000), seed=7100 + i, pretty_bias=0.8)) for i in range(4)]
    docs += [O.jsonexample(f) for f in ("twitter.json", "citm_catalog.json", "amazon_cellphones.ndjson")]
    checked, with_errors = 0, 0
    for d in docs:
        r = port.stage1(d)
        assert r.err == 0
        want = whole(port, d, r.idx, r.n)
        with_errors += want[0] not in (0, 1)
        for kind in ("lf", "quote", "operator", "ws"):
            for nshards in (2, 4, 7):
                cuts = clean_cuts(port, d, rng, nshards, kind)
                if len(cuts) < 3:
                    continue
                assert same(sharded(emu, d, r.idx, r.n, cuts), want), (d[:60], kind, cuts)
                checked += 1
    assert checked > 150 and with_errors >= 8


def test_errors_in_several_shards_fold_to_the_first(emu):  # noqa: F811
    """token errors planted in chosen shards: the earliest shard's first error is the document's"""
    port = O.Port()
    rng = random.Random(corpus.SEED ^ 0xE77)
    rows = [b'{"a": ' + str(rng.randrange(10 ** 6)).encode() + b', "s": "' + TF.string_body(rng, bad_rate=0.0)[0] + b'", "t": true}' for _ in range(400)]
    for plant in ((1, 3), (3,), (0, 2, 3), ()):
        body = list(rows)
        for s in plant:
            k = s * 100 + rng.randrange(100)
            body[k] = body[k].replace(b"true", rng.choice([b"tru", b"nul", b"-x", b"1e", b'"\\q"']))
        d = b"\n".join(body) + b"\n"
        r = port.stage1(d)
        want = whole(port, d, r.idx, r.n)
        assert (want[0] not in (0, 1)) == bool(plant)
        offs = np.cumsum([0] + [len(x) + 1 for x in body])
        cuts = [int(offs[100 * k]) for k in range(4)] + [len(d)]
        assert same(sharded(emu, d, r.idx, r.n, cuts), want), plant


def test_edge_shards(emu):  # noqa: F811
    port = O.Port()
    rng = random.Random(corpus.SEED ^ 0xED6)
    # shards with no structurals: a whitespace run cut at both ends
    d = b'[1, "a",' + b" " * 5000 + b"\n" * 300 + b'"b", 2.5e3,\n' + b"\t" * 700 + b"null]"
    r = port.stage1(d)
    want = whole(port, d, r.idx, r.n)
    for cuts in ([0, 10, 2000, 5100, len(d)], [0, 9, 5301, 5305, 5308, 5320, 5325, len(d)], [0, 5400, 5700, 6000, len(d)]):
        assert all(_state(port, d[:c]) == 0 for c in cuts[1:-1])
        assert same(sharded(emu, d, r.idx, r.n, cuts), want), cuts
    # strings longer than the lane budget (96 bytes: the kernels hand them to a whole warp) ending right before a cut
    for _ in range(20):
        parts, cuts = [], [0]
        doc = bytearray(b"[")
        for _ in range(rng.randrange(3, 9)):
            body = TF.long_body(rng, rng.choice([97, 200, 513, 3000, 20000]), rng.choice([0.0, 0.05, 0.3]))
            doc += b'"' + body + b'"'
            cuts.append(len(doc))
            doc += rng.choice([b",", b" , ", b",\n"]) + str(rng.randrange(10 ** 9)).encode() + b","
            parts.append(body)
        doc += b"0]"
        d = bytes(doc)
        cuts.append(len(d))
        assert all(_state(port, d[:c]) == 0 for c in cuts[1:-1])
        r = port.stage1(d)
        assert r.err == 0
        assert same(sharded(emu, d, r.idx, r.n, cuts), whole(port, d, r.idx, r.n))


def test_dirty_cuts_give_other_tokens(emu):  # noqa: F811
    """the precondition is needed: a cut inside a string or a number, state != 0, changes the tokens"""
    port = O.Port()
    d = b'[12345678, "abc def ghi", 3.25, "x\\"y", true]'
    r = port.stage1(d)
    want = whole(port, d, r.idx, r.n)
    for at in (d.index(b"5678"), d.index(b"def"), d.index(b"25,"), d.index(b'\\"') + 1, d.index(b"rue")):
        assert _state(port, d[:at]) != 0
        got = sharded(emu, d, r.idx, r.n, [0, at, len(d)])
        assert not same(got, want), at
