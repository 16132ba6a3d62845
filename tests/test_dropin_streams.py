"""Streams through the drop-in path: dom::parser::parse_many and ondemand::parser::iterate_many of the UNMODIFIED
simdjson API, in every stream format, walked to their end with the "b200" plug-in active and with a CPU implementation
active.  The harness (simdjson_b200/plugin/dropin_harness.cpp) records, per iterator position, the error,
current_index(), source() and the document's compact JSON, then the stream's truncated_bytes() and size_in_bytes(): the
document boundaries that document_stream reads back out of the plug-in's index array (structural_indexes[n] and
[n + 1]) show up there even when the documents themselves are right.  Two walks are equal when their record blobs are
byte-identical; the decoded records only serve the messages and the pinning tests.

  a  the harness, on the CPU implementation, against records computed here from the json module and known offsets
  b  plug-in vs CPU: both APIs, every format, threaded or not, batch sizes from MINIMAL_BATCH_SIZE up, several corpora
  c  batch windows cut right before, on and after every hazard byte of a small stream (backslash, quote, UTF-8 lead and
     continuation, RS, root comma, digit, atom), then the stream repeated so that later windows land at other phases
  d  streams with errors, every record the API still yields after the first error included
  e  one dom::parser reused across documents of growing and shrinking sizes with failing documents between them
"""
import ctypes as C
import json
import math
import os
import random
import struct

import numpy as np
import pytest

import oracle_lib as O
import token_fuzz as TF
from simdjson_b200 import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "simdjson_b200", "plugin", "libsimdjson_b200.so")
needs_plugin = pytest.mark.skipif(not os.path.exists(PLUGIN), reason="plug-in not built (needs the reference headers)")

# simdjson error codes (include/simdjson/error.h)
SUCCESS, CAPACITY, TAPE_ERROR, UTF8_ERROR, EMPTY, UNESCAPED_CHARS, UNCLOSED_STRING = 0, 1, 3, 11, 13, 14, 15
MINIMAL_BATCH_SIZE, DEFAULT_BATCH_SIZE = 32, 1000000
NONE, OUT_OF_RANGE = (1 << 64) - 1, (1 << 64) - 2

# stream formats of the harness: simdjson::stream_format in order, then ondemand's deprecated allow_comma_separated
WS, SEQ, COMMA, ARRAY, ALLOW_COMMA = 0, 1, 2, 3, 4
FORMAT_NAMES = {WS: "whitespace", SEQ: "json_sequence", COMMA: "comma_delimited", ARRAY: "comma_delimited_array", ALLOW_COMMA: "allow_comma_separated"}
DOM_FORMATS = (WS, SEQ, COMMA, ARRAY)
OD_FORMATS = (WS, SEQ, COMMA, ARRAY, ALLOW_COMMA)
API_FORMATS = [("dom", f) for f in DOM_FORMATS] + [("ondemand", f) for f in OD_FORMATS]
API_FORMAT_IDS = ["%s-%s" % (a, FORMAT_NAMES[f]) for a, f in API_FORMATS]
TRAILER = struct.Struct("<iQiQQ")
PAD_FILLS = (0x22, 0x5C, 0x31, 0xFF, 0x5D)


class Walks:
    def __init__(self):
        L = C.CDLL(PLUGIN)
        u8, sz, ull = C.c_void_p, C.c_size_t, C.POINTER(C.c_ulonglong)
        for f in (L.dropin_stream_dom, L.dropin_stream_ondemand):
            f.restype = C.c_int
            f.argtypes = [C.c_int, u8, sz, sz, C.c_int, C.c_int, C.c_int, sz, C.c_char_p, sz, C.POINTER(sz), ull]
        L.dropin_dom_sequence.restype = C.c_int
        L.dropin_dom_sequence.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.POINTER(sz), sz, sz, C.c_char_p, sz, C.POINTER(sz), ull]
        self.L = L

    @staticmethod
    def _call(fn, cap):
        """fn(out, cap, out_len) -> rc; grows the output once if the records did not fit"""
        while True:
            out, ol = C.create_string_buffer(cap), C.c_size_t(0)
            rc = fn(out, cap, ol)
            if ol.value <= cap:
                return rc, out.raw[: ol.value]
            cap = ol.value

    def stream(self, api, use_b200, data, batch, fmt, threaded=0, pad_fill=0x22, max_records=None):
        """one walk: (record blob, stage-1 calls sent to the GPU)"""
        a = np.frombuffer(bytes(data), dtype=np.uint8)
        fn = self.L.dropin_stream_dom if api == "dom" else self.L.dropin_stream_ondemand
        mr = len(a) + 8 if max_records is None else max_records
        calls = C.c_ulonglong(0)
        rc, blob = self._call(lambda out, cap, ol: fn(use_b200, a.ctypes.data, len(a), batch, fmt, threaded, pad_fill, mr, out, cap,
                                                      C.byref(ol), C.byref(calls)), 3 * len(a) + 4096)
        assert rc == 0, (api, fmt)
        return blob, calls.value

    def sequence(self, use_b200, docs, initial_capacity=0):
        arrs = [np.frombuffer(bytes(d), dtype=np.uint8) if len(d) else np.zeros(1, dtype=np.uint8) for d in docs]
        ptrs = (C.c_void_p * len(docs))(*[a.ctypes.data for a in arrs])
        lens = (C.c_size_t * len(docs))(*[len(d) for d in docs])
        calls = C.c_ulonglong(0)
        rc, blob = self._call(lambda out, cap, ol: self.L.dropin_dom_sequence(use_b200, ptrs, lens, len(docs), initial_capacity, out, cap,
                                                                              C.byref(ol), C.byref(calls)),
                              2 * sum(len(d) for d in docs) + 4096)
        assert rc == 0
        return blob, calls.value


def decode(blob, api):
    """records [(error, current_index, source, json)] (ondemand: json = (to_json_string error, text)) and the trailer"""
    body, trailer = blob[: -TRAILER.size], blob[-TRAILER.size:]
    pos, recs = 0, []

    def i32():
        nonlocal pos
        v = struct.unpack_from("<i", body, pos)[0]
        pos += 4
        return v

    def u64():
        nonlocal pos
        v = struct.unpack_from("<Q", body, pos)[0]
        pos += 8
        return v

    def field():
        nonlocal pos
        n = u64()
        if n in (NONE, OUT_OF_RANGE):
            return None if n == NONE else "out of range"
        v = body[pos: pos + n]
        pos += n
        return v

    while pos < len(body):
        err, idx, src = i32(), u64(), field()
        js = field() if api == "dom" else (i32(), field())
        recs.append((err, idx, src, js))
    create_err, n, cap_hit, truncated, size = TRAILER.unpack(trailer)
    assert n == len(recs)
    return dict(records=recs, create_err=create_err, cap_hit=cap_hit, truncated=None if truncated == NONE else truncated,
                size=None if size == NONE else size)


def decode_sequence(blob):
    pos, out = 0, []
    while pos < len(blob):
        err, n = struct.unpack_from("<iQ", blob, pos)
        pos += 12
        if n == NONE:
            out.append((err, None))
        else:
            out.append((err, blob[pos: pos + n]))
            pos += n
    return out


@pytest.fixture(scope="module")
def w():
    return Walks()


def _first_difference(g, c, api):
    dg, dc = decode(g, api), decode(c, api)
    for i, (rg, rc) in enumerate(zip(dg["records"], dc["records"])):
        if rg != rc:
            return "record %d: plug-in %r, cpu %r" % (i, _short(rg), _short(rc))
    if len(dg["records"]) != len(dc["records"]):
        return "records: plug-in %d, cpu %d (last cpu %r)" % (len(dg["records"]), len(dc["records"]), _short(dc["records"][-1:]))
    return "trailer: plug-in %r, cpu %r" % ({k: v for k, v in dg.items() if k != "records"}, {k: v for k, v in dc.items() if k != "records"})


def _short(x):
    s = repr(x)
    return s if len(s) < 300 else s[:300] + "..."


def effective_len(data, fmt):
    """the length document_stream walks: parse_many / iterate_many drop a BOM and, for comma_delimited_array, the brackets
    with the JSON whitespace around them"""
    n = len(data)
    start = 3 if data[:3] == b"\xef\xbb\xbf" else 0
    if fmt == ARRAY:
        ws = b" \t\n\r"
        while start < n and data[start] in ws:
            start += 1
        start += 1
        while n > start and data[n - 1] in ws:
            n -= 1
        n -= 1
    return max(0, n - start)


def compare(w, api, data, batch, fmt, threaded, pad_fill=0x22, ctx=()):
    """plug-in and CPU walks of one stream must give byte-identical records; a walk that reaches the end of the stream
    sent every window to the GPU.  Returns the decoded CPU records."""
    c, _ = w.stream(api, 0, data, batch, fmt, threaded, pad_fill)
    g, calls = w.stream(api, 1, data, batch, fmt, threaded, pad_fill)
    where = (api, FORMAT_NAMES[fmt], "threaded" if threaded else "unthreaded", "batch", batch, "len", len(data)) + tuple(ctx)
    assert g == c, (where, _first_difference(g, c, api))
    d = decode(c, api)
    assert not d["cap_hit"], where
    recs = d["records"]
    consumed = d["create_err"] == SUCCESS and (not recs or recs[-1][0] == SUCCESS)
    eff = effective_len(data, fmt)
    if consumed and eff > 0:
        want = math.ceil(eff / max(batch, MINIMAL_BATCH_SIZE))
        assert calls >= want, (where, calls, want)
    return d


# =========================================================================== a: the harness itself, CPU only
def _expected(docs, fmt, lead=b"", trail=b""):
    """stream bytes and the records a correct walk yields: offsets computed from the joined pieces, JSON from the json
    module (documents here are ASCII, integers, no escapes: the compact form is unique)"""
    out = bytearray(lead)
    if fmt == ARRAY:
        out += b"["
    base = len(out)
    recs = []
    for i, (text, tail) in enumerate(docs):
        if fmt == SEQ:
            out += b"\x1e"
        at = len(out) - base
        out += text
        compact = json.dumps(json.loads(text), separators=(",", ":")).encode()
        recs.append((at, text.strip(), compact))
        out += tail
    if fmt == ARRAY:
        out += b"]"
    out += trail
    return bytes(out), recs


PIN_DOCS = [(b'{"a":1}', b" "), (b"[1, 2,3]", b"\n"), (b'"x"', b" "), (b"12", b"  "), (b"true", b"\t"), (b'{"b":[true,false,null]}', b" "),
            (b"[]", b" "), (b"-7", b"\n")]
PIN_SEPARATORS = {WS: None, SEQ: b"\n", COMMA: b",", ARRAY: b",", ALLOW_COMMA: b","}


def _pin_stream(fmt, containers_only=False):
    # (ondemand: after to_json_string() of a scalar root the reference's iterator also steps over the next document, on
    # every implementation; the scalar streams are compared with the CPU in parts b-d instead of being pinned here)
    pin = [(t, tail) for t, tail in PIN_DOCS if not containers_only or t[:1] in b"[{"]
    sep = PIN_SEPARATORS[fmt]
    docs = [(t, tail if sep is None else (tail + sep if i + 1 < len(pin) else tail)) for i, (t, tail) in enumerate(pin)]
    if fmt == SEQ:
        docs = [(t, b"\n") for t, _ in pin]
    return _expected(docs, fmt, lead=b"\xef\xbb\xbf" if fmt == COMMA else b"", trail=b" " if fmt == ARRAY else b"")


@needs_plugin
@pytest.mark.parametrize("api,fmt", API_FORMATS, ids=API_FORMAT_IDS)
def test_harness_records_known_stream(w, api, fmt):
    """no GPU: the CPU implementation through the new entry points yields the documents, offsets, sources and JSON
    computed here, at the default batch size and at batch sizes that cut the stream into many windows"""
    data, want = _pin_stream(fmt, containers_only=api == "ondemand")
    eff = effective_len(data, fmt)
    for batch in (DEFAULT_BATCH_SIZE, 64, MINIMAL_BATCH_SIZE, 5):
        for threaded in (0, 1):
            blob, calls = w.stream(api, 0, data, batch, fmt, threaded)
            d = decode(blob, api)
            assert calls == 0
            assert (d["create_err"], d["cap_hit"], d["size"]) == (SUCCESS, 0, eff), (batch, d)
            if fmt == WS:
                # (in the delimited formats the final window's truncated_bytes() is len minus whatever index word the
                # separator filter left at [n], a value this test does not restate: part b compares it with the CPU)
                assert d["truncated"] == 0, (batch, d)
            got = d["records"]
            assert len(got) == len(want), (batch, threaded, got)
            for (err, idx, src, js), (at, text, compact) in zip(got, want):
                assert (err, idx) == (SUCCESS, at), (batch, threaded, err, idx, at)
                if api == "dom":
                    assert (src, js) == (text, compact), (batch, threaded, src, js)
                else:
                    # (to_json_string gives the document's own bytes, whitespace inside included, and in an RS stream
                    # the separator bytes up to the next document as well)
                    assert js[0] == SUCCESS and js[1].rstrip(b" \t\n\r\x1e,") == text, (batch, threaded, js)
                    assert src == text, (batch, threaded, src, text)


@needs_plugin
@pytest.mark.parametrize("api", ["dom", "ondemand"])
def test_harness_records_truncation_and_capacity(w, api):
    """no GPU: a stream cut inside its last document ends after the complete ones with truncated_bytes() = the bytes of
    the cut document; a document longer than the batch ends the walk with CAPACITY and truncated_bytes() = len -
    batch_start; an empty input yields nothing; comma_delimited_array without its brackets fails at creation"""
    data = b'{"a":1} [1,2] {"b":[1,'
    d = decode(w.stream(api, 0, data, DEFAULT_BATCH_SIZE, WS)[0], api)
    assert [(r[0], r[1]) for r in d["records"]] == [(SUCCESS, 0), (SUCCESS, 8)]
    assert d["truncated"] == len(b'{"b":[1,'), d
    big = b"[" + b"1," * 40 + b"1]"
    data = b"[0] [1]\n" + big + b" [2]"
    d = decode(w.stream(api, 0, data, 64, WS)[0], api)
    assert [r[0] for r in d["records"]] == [SUCCESS, SUCCESS, CAPACITY], d
    assert d["truncated"] == len(data) - data.index(big), d
    for fmt in DOM_FORMATS:
        d = decode(w.stream(api, 0, b"", 64, fmt)[0], api) if fmt != ARRAY else None
        if d is not None:
            assert d["records"] == [] and d["create_err"] == SUCCESS, (fmt, d)
    for bad in (b"{}", b" [1],[2", b"1,2]", b"", b"  ", b"[", b"]"):
        d = decode(w.stream(api, 0, bad, 64, ARRAY)[0], api)
        assert d["create_err"] == TAPE_ERROR and d["records"] == [], (bad, d)


@needs_plugin
def test_harness_sequence_records(w):
    """no GPU: dropin_dom_sequence records each parse's error and compact JSON in order"""
    docs = [b"1", b'{"a": [1, 2]}', b'["\xff"]', b'{"a":1', b"", b" [ true ] "]
    got = decode_sequence(w.sequence(0, docs)[0])
    assert got == [(SUCCESS, b"1"), (SUCCESS, b'{"a":[1,2]}'), (UTF8_ERROR, None), (TAPE_ERROR, None), (EMPTY, None), (SUCCESS, b"[true]")], got
    assert decode_sequence(w.sequence(0, docs, initial_capacity=4)[0]) == got


# =========================================================================== inputs
def join(docs, fmt):
    """documents (bytes) as a stream of the given format"""
    if fmt == WS:
        return b"".join(d + b"\n" for d in docs)
    if fmt == SEQ:
        return b"".join(b"\x1e" + d + b"\n" for d in docs)
    if fmt in (COMMA, ALLOW_COMMA):
        return b",".join(docs)
    return b"[" + b",".join(docs) + b"]"


def ndjson_docs(nbytes, seed):
    return [r for r in bytes(corpus.ndjson_rows(nbytes, seed=seed)).split(b"\n") if r]


def amazon_docs():
    return [r for r in O.jsonexample("amazon_cellphones.ndjson").split(b"\n") if r.strip()]


def tile_docs(nbytes):
    small = [b"1", b"-2.5e3", b"true", b"false", b"null", b'"s"', b'"a\\"b"', b"[]", b"{}", b"[[]]", b'{"k":{}}', b"[1,[2,[3]]]", b'"\xc3\xa9"',
             b'{"a":"x","b":[null]}']
    return [d for d in bytes(corpus.tile_documents(small, nbytes, sep=b"\n")).split(b"\n") if d]


def fuzz_docs(w, seed, count, max_len=None):
    """rows with escapes and multi-byte UTF-8, each accepted by the CPU implementation on its own (the json module also
    accepts documents simdjson rejects, such as integers past 64 bits).  max_len keeps rows shorter than small batches,
    and arrays or objects only, since a window cutting a root scalar ends the stream"""
    rng = random.Random(seed)
    out = []
    while len(out) < count:
        cand = []
        while len(cand) < 2 * (count - len(out)):
            r = rng.random()
            if r < 0.5:
                body, bad = TF.string_body(rng, bad_rate=0.0)
                if not bad:
                    cand.append(b'["' + body + b'"]' if max_len is not None or rng.random() < 0.5 else b'"' + body + b'"')
            elif r < 0.8:
                cand.append(TF.wrap_scalar(TF.scalar_token(rng), rng)[0])
            else:
                body, bad = TF.string_body(rng, bad_rate=0.0, maxlen=64)
                if not bad:
                    cand.append(b'{"k\\n":"' + body + b'","v":[1,-0.5,"\xe2\x82\xac",{"\xf0\x9f\x98\x80":true}]}')
            if max_len is not None and cand and len(cand[-1]) > max_len:
                cand.pop()
        out += cpu_accepted(w, cand)[: count - len(out)]
    return out


def cpu_accepted(w, docs):
    """the documents dom::parser::parse accepts with the CPU implementation active"""
    recs = decode_sequence(w.sequence(0, docs)[0])
    return [d for d, (err, _) in zip(docs, recs) if err == SUCCESS]


def hostile_streams(fmt):
    """the separators' own edge cases for one format"""
    if fmt == SEQ:
        return [b"\x1e1\n\x1e\"a\"\n\x1etrue\n\x1e-0.5\n\x1e[1]\n", b"\x1e\x1e\x1e{}\n\x1e\n\x1e[]", b"\x1e{\"a\":1}\x1e[2]\x1e3\x1e\"x\"",
                b"\x1e 1 \n\x1e\n\n\x1e null", b"[1]\n\x1e[2]\n", b"\x1e" * 5 + b"[0]" + b"\x1e" * 20 + b"{}"]
    if fmt in (COMMA, ALLOW_COMMA):
        return [b"1,2,3,", b"[1],,[2]", b'{"a":[1,2]},"x",true,null,', b" 1 , 2 ,[3, 4] , {\"b\":5} ", b",[1]", b"1," * 30 + b"1"]
    if fmt == ARRAY:
        return [b"[1,2,3]", b" \n[ [1] , {\"a\":[2,3]} , \"x\" ]\r\n", b"[1,]", b"[[],[]]", b"[" + b"{},"  * 30 + b"{}]"]
    return [b"1 2 3", b'{"a":1}{"b":2}[3]"x"4', b"  \n\t[1]\r\n  ", b"true false null"]


def blank_streams(fmt):
    # (RS-only streams stay within one window of MINIMAL_BATCH_SIZE bytes: given a longer one, the reference's
    # document_stream::start() never returns in json_sequence mode whatever the implementation -- a partial window
    # without a record leaves next_batch_start() where the window began)
    return [b"", b" ", b" \n\t\r" * 20, b"\x1e", b"\x1e" * 31, b"\x1e\n" * 15, b"," if fmt in (COMMA, ALLOW_COMMA) else b""]


def random_batches(seed, count, lo=33, hi=3000):
    rng = random.Random(seed)
    return [rng.randrange(lo, hi) for _ in range(count)]


SMALL_BATCHES = (MINIMAL_BATCH_SIZE, 33, 63, 64, 65, 127)
LARGE_BATCHES = (4096, DEFAULT_BATCH_SIZE)


def whole_from(docs):
    """a batch size from which every window holds at least one whole document and the separators around it, so a walk
    of valid documents yields all of them"""
    return 2 * max(len(d) for d in docs) + 8


class Corpus:
    """one stream: its bytes, the batch sizes it is walked at, and for streams of valid documents their count and
    the batch size from which a dom walk must yield every one of them"""
    def __init__(self, name, data, batches, docs=None):
        self.name, self.data, self.batches = name, data, tuple(batches)
        self.ndocs = None if docs is None else len(docs)
        self.whole_from = None
        if docs is not None:
            # (a root scalar that a window cuts, "tr|ue", is an atom error in the reference whatever the implementation:
            # streams with root scalars are only whole when they fit in one window)
            scalars = any(d[:1] not in (b"[", b"{") for d in docs)
            self.whole_from = len(data) if scalars else whole_from(docs)


def corpora(w, fmt):
    """the streams of one format.  Rows longer than the small batches are walked from whole_from up (below it every
    walk ends at the first long row); batch sizes below 4096 only on streams of at most 64 KiB."""
    small = SMALL_BATCHES + tuple(random_batches(1000 + fmt, 3)) + LARGE_BATCHES

    def valid(name, docs, batches, bom=False):
        return Corpus(name, (b"\xef\xbb\xbf" if bom else b"") + join(docs, fmt), batches, docs)

    def long_rows(name, docs, seed, extra=(), n_random=2):
        lo = whole_from(docs)
        return valid(name, docs, (lo, lo + 1) + tuple(random_batches(seed, n_random, lo, 4 * lo)) + tuple(extra) + LARGE_BATCHES)

    out = [
        long_rows("ndjson", cpu_accepted(w, ndjson_docs(48 << 10, 11)), 2000 + fmt),
        long_rows("ndjson-large", cpu_accepted(w, ndjson_docs(1 << 20, 12)), 3000 + fmt, (65536 + 7,), n_random=0),
        long_rows("amazon", amazon_docs(), 4000 + fmt, (10007,)),
        long_rows("fuzz", fuzz_docs(w, fmt, 400), 5000 + fmt),
        valid("fuzz-short", fuzz_docs(w, 10 + fmt, 800, max_len=30), small),
        valid("tiles", tile_docs(16 << 10), small),
        valid("bom", fuzz_docs(w, 50 + fmt, 200, max_len=30), small, bom=True),
    ]
    out += [Corpus("hostile%d" % i, s, small) for i, s in enumerate(hostile_streams(fmt))]
    out += [Corpus("blank%d" % i, s, (MINIMAL_BATCH_SIZE, 33, 64, DEFAULT_BATCH_SIZE)) for i, s in enumerate(blank_streams(fmt))]
    return out


def assert_whole(d, c, batch, where):
    """a dom walk of valid documents at a batch of at least whole_from yields all of them, without error, to the end"""
    if c.ndocs is None or batch < c.whole_from:
        return
    errs = [r[0] for r in d["records"]]
    assert len(errs) == c.ndocs and not any(errs), (where, c.name, batch, len(errs), c.ndocs, [e for e in errs if e][:1])


@needs_plugin
@pytest.mark.parametrize("fmt", DOM_FORMATS, ids=lambda f: FORMAT_NAMES[f])
def test_corpora_are_walked_whole(w, fmt):
    """no GPU: every corpus of valid documents is yielded whole by the CPU implementation at the default batch size and
    from whole_from up, so a generator that produced a document simdjson rejects cannot silently cut the comparisons short"""
    for c in corpora(w, fmt):
        if c.ndocs is None:
            continue
        assert c.ndocs >= 60 and c.whole_from <= DEFAULT_BATCH_SIZE, (c.name, c.ndocs, c.whole_from)
        for batch in sorted({b for b in c.batches if b >= c.whole_from}):
            assert_whole(decode(w.stream("dom", 0, c.data, batch, fmt)[0], "dom"), c, batch, FORMAT_NAMES[fmt])


# =========================================================================== b: plug-in vs CPU
@needs_plugin
@pytest.mark.gpu
@pytest.mark.parametrize("threaded", [0, 1])
@pytest.mark.parametrize("api,fmt", API_FORMATS, ids=API_FORMAT_IDS)
def test_streams_match_cpu(w, api, fmt, threaded):
    for k, c in enumerate(corpora(w, fmt)):
        for batch in c.batches:
            d = compare(w, api, c.data, batch, fmt, threaded, PAD_FILLS[k % len(PAD_FILLS)], ctx=(c.name,))
            if api == "dom":
                assert_whole(d, c, batch, (api, FORMAT_NAMES[fmt], threaded))


# =========================================================================== c: cuts at every hazard
HAZARD_DOCS = [b'{"k":"a\\"b\\\\","u":"\xc3\xa9\xe2\x82\xac\xf0\x9f\x98\x80"}', b"[12345,-6.75e+10,true,false,null]", b'"\\u00e9\\n\xe4\xb8\xad"',
               b"98765", b'["\\\\\\"",{"\xc3\xbc":[]}]', b"null", b'{"a":[1,{"b":"c,d\\u001e"}]}', b"-0.125", b"true"]


def hazards(stream, start):
    """offsets (relative to where document_stream starts) of the bytes where a window end is most likely to go wrong"""
    out = []
    for i in range(start, len(stream)):
        c = stream[i]
        if c in b'\\"' or c >= 0x80 or c == 0x1E or c in b"0123456789-+.eE" or c in b"truefalsn":
            out.append(i - start)
        elif c == 0x2C:
            out.append(i - start)
    return out


@needs_plugin
@pytest.mark.gpu
@pytest.mark.parametrize("api,fmt", API_FORMATS, ids=API_FORMAT_IDS)
def test_windows_cut_at_hazards(w, api, fmt):
    once = join(HAZARD_DOCS, fmt)
    start = 1 if fmt == ARRAY else 0
    hs = [h for h in hazards(once, start) if h >= 33]
    assert len(hs) > 60
    for reps in (1, 3):
        data = join(HAZARD_DOCS * reps, fmt)
        for i, h in enumerate(hs):
            for batch in (h - 1, h, h + 1):
                compare(w, api, data, batch, fmt, (i + batch) % 2, ctx=("hazard", h, "byte", once[start + h: start + h + 1], "reps", reps))


# =========================================================================== d: streams with errors
def join_then(docs, last, fmt):
    """the stream of docs followed by the raw bytes `last` where one more document would go"""
    if fmt == WS:
        return join(docs, fmt) + last
    if fmt == SEQ:
        return join(docs, fmt) + b"\x1e" + last
    if fmt in (COMMA, ALLOW_COMMA):
        return join(docs, fmt) + b"," + last
    return b"[" + b",".join(docs) + b"," + last + b"]"


def error_streams(fmt):
    good = [b'{"a":1}', b"[1,2]", b'"x"', b"12", b"[true]"]
    big = b'{"big":[' + b",".join(b'"%05d"' % i for i in range(700)) + b"]}"
    out = {
        "utf8-2nd-of-5": join([good[0], b'["\xff"]'] + good[2:], fmt),
        "utf8-2nd-of-5-in-string": join([good[0], b'{"s":"a\xc3(b"}'] + good[2:], fmt),
        "unescaped-control": join(good[:2] + [b'["a\x01b"]'] + good[2:], fmt),
        "unclosed-string-end": join_then(good, b'"abc', fmt),
        "unclosed-string-middle": join(good[:2] + [b'["abc'] + good[2:], fmt),
        "larger-than-batch": join(good[:3] + [big] + good[3:], fmt),
        "truncated-last": join_then(good, b'{"b":[1,', fmt),
        "trailing-garbage": join_then(good, b"xyz @!", fmt),
        "bad-atom": join(good[:2] + [b"[tru]", b"nul"] + good[2:], fmt),
        "unbalanced": join(good[:2] + [b"[1,2}", b"]"] + good[2:], fmt),
    }
    if fmt == ARRAY:
        out["no-open-bracket"] = b",".join(good) + b"]"
        out["no-close-bracket"] = b"[" + b",".join(good) + b",3"
    return out


@needs_plugin
@pytest.mark.gpu
@pytest.mark.parametrize("api,fmt", API_FORMATS, ids=API_FORMAT_IDS)
def test_streams_with_errors(w, api, fmt):
    for name, data in error_streams(fmt).items():
        for batch in (MINIMAL_BATCH_SIZE, 40, 64, 100, 4096, DEFAULT_BATCH_SIZE):
            for threaded in (0, 1):
                d = compare(w, api, data, batch, fmt, threaded, ctx=(name,))
                if name.startswith("no-") and fmt == ARRAY:
                    assert d["create_err"] == TAPE_ERROR and d["records"] == [], (name, d)
                if name == "larger-than-batch" and batch == 4096:
                    # (ondemand reports the window cut inside the document as CAPACITY or TAPE_ERROR by format)
                    assert d["records"][-1][0] == CAPACITY if api == "dom" else d["records"][-1][0] != SUCCESS, (name, d["records"][-1])
                if name == "utf8-2nd-of-5" and batch == DEFAULT_BATCH_SIZE:
                    assert any(r[0] == UTF8_ERROR for r in d["records"]), (name, d)


@needs_plugin
@pytest.mark.gpu
@pytest.mark.parametrize("api", ["dom", "ondemand"])
def test_document_larger_than_batch_truncates_from_its_window(w, api):
    """CAPACITY on a window that starts inside the stream: truncated_bytes() = len - batch_start, batch_start being where
    the window holding the large document begins (4096 bytes of small rows, then the large document)"""
    small = b"".join(b'[%d]\n' % i for i in range(300))
    small += b" " * (4096 - len(small))
    big = b'{"big":"' + b"x" * 6000 + b'"}'
    data = small + big + b"\n[1]\n"
    for threaded in (0, 1):
        d = compare(w, api, data, 4096, WS, threaded)
        assert d["records"][-1][0] == CAPACITY and len(d["records"]) == 301, d["records"][-2:]
        # (the first window ends where the large document starts: the second begins there)
        assert d["truncated"] == len(data) - len(small), (d["truncated"], len(data) - len(small))


# =========================================================================== e: one parser, many documents
def _sized(n, seed):
    if n == 1:
        return b"1"
    if n == 16:
        return b'{"a":[1,2,3,4]} '
    doc = bytes(corpus.random_json(n, seed=seed))
    assert len(doc) == n
    return doc


BAD_DOCS = [b'["\xff"]', b'{"a":1', b'["a\x01b"]', b""]


@needs_plugin
@pytest.mark.gpu
@pytest.mark.parametrize("initial_capacity", [0, 1000])
def test_parser_reuse_across_sizes(w, initial_capacity):
    """capacity growth (set_capacity re-pins the new index array), smaller documents after larger ones (the words past
    n are stale) and failing documents between good ones, through one dom::parser"""
    sizes = (1, 64, 4096, 1 << 20, 16, 3 << 20, 100)
    docs = []
    for i, n in enumerate(sizes):
        docs.append(_sized(n, 70 + i))
        if i + 1 < len(sizes):
            docs.append(BAD_DOCS[i % len(BAD_DOCS)])
    c, _ = w.sequence(0, docs, initial_capacity)
    g, calls = w.sequence(1, docs, initial_capacity)
    dc = decode_sequence(c)
    assert g == c, [(i, x, y) for i, (x, y) in enumerate(zip(decode_sequence(g), dc)) if x != y][:1]
    assert [e for e, _ in dc] == [SUCCESS, UTF8_ERROR, SUCCESS, TAPE_ERROR, SUCCESS, UNESCAPED_CHARS, SUCCESS, EMPTY, SUCCESS, UTF8_ERROR,
                                  SUCCESS, TAPE_ERROR, SUCCESS], dc
    assert calls >= len(docs) - 1  # every non-empty document went through the GPU's stage 1
