"""ctypes bindings for the two stage-2 grammar checkers (test infrastructure only; recipe: oracle/grammar.mk), and the
cases the document-error tests share.

  Grammar    : oracle/libsj_grammar_oracle.so    -- sjo_document_errors, our restatement of walk_document over the
                                                    oracle's tokens (always built)
  RefGrammar : oracle/_ref/libsj_ref_grammar.so  -- the unmodified reference's parse and stage2_next (may be absent)
"""
import ctypes as C
import json
import os
import random
import subprocess

import numpy as np

import oracle_lib as O
import pointer_oracle as PO

ORACLE_DIR = O.ORACLE_DIR
MAKEFILE = os.path.join(ORACLE_DIR, "grammar.mk")
GRAM_SO = os.path.join(ORACLE_DIR, "libsj_grammar_oracle.so")
REF_GRAM_SO = os.path.join(ORACLE_DIR, "_ref", "libsj_ref_grammar.so")
GOLDEN = os.path.join(os.path.dirname(ORACLE_DIR), "tests", "golden", "document_errors.json")

TAPE_ERROR, DEPTH_ERROR, STRING_ERROR, NUMBER_ERROR, EMPTY, UNEXPECTED_ERROR = 3, 4, 5, 9, 13, 24
NONE = 0xFFFFFFFF


def _ptr(a, t=C.c_uint8):
    return a.ctypes.data_as(C.POINTER(t))


class Grammar:
    """sjo_document_errors over the tokens of oracle_lib.Port"""

    def __init__(self):
        if not os.path.exists(GRAM_SO) or os.path.getmtime(GRAM_SO) < os.path.getmtime(os.path.join(ORACLE_DIR, "sj_grammar_oracle.c")):
            subprocess.check_call(["make", "-f", MAKEFILE, GRAM_SO], stdout=subprocess.DEVNULL)
        L = C.CDLL(GRAM_SO)
        L.sjo_document_errors.restype = C.c_int
        L.sjo_document_errors.argtypes = [C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32, C.c_size_t,
                                          C.POINTER(C.c_int32), C.POINTER(C.c_uint32)]
        self.L = L
        self.port = O.Port()

    def tokens(self, buf):
        """stage 1 (regular) and tokens: (stage1 result, types, payloads); None when stage 1 fails"""
        r = self.port.stage1(buf)
        if r.err != 0:
            return None
        tw = self.port.tokens(buf, r.idx, r.n)
        return r, tw[1], tw[2]

    def errors(self, types, payload, starts=None, max_depth=1024):
        """per document (error int32[D], index uint32[D]); starts None: one document"""
        n = len(types)
        t = np.ascontiguousarray(types, dtype=np.uint8) if n else np.zeros(1, dtype=np.uint8)
        p = np.ascontiguousarray(payload, dtype=np.uint64) if n else np.zeros(1, dtype=np.uint64)
        D = 1 if not starts else len(starts)
        st = np.ascontiguousarray(starts if starts else [0], dtype=np.uint32)
        err = np.zeros(D, dtype=np.int32)
        idx = np.zeros(D, dtype=np.uint32)
        self.L.sjo_document_errors(_ptr(t), _ptr(p, C.c_uint64), n, _ptr(st, C.c_uint32) if starts else None, len(starts) if starts else 0, max_depth,
                                   _ptr(err, C.c_int32), _ptr(idx, C.c_uint32))
        return err, idx

    def stream(self, buf, max_depth=1024, table=True):
        """stage 1, tokens, the document starts and the verdicts of a stream (None when stage 1 fails)"""
        tk = self.tokens(buf)
        if tk is None:
            return None
        r, types, pay = tk
        starts = PO.document_starts(buf, r.idx, r.n) if table else None
        err, idx = self.errors(types, pay, starts, max_depth)
        return r, types, pay, starts, err, idx


def have_ref():
    return os.path.exists(REF_GRAM_SO) and O.have_ref()


class RefGrammar:
    """the unmodified reference: dom::parser::parse, and stage2_next from each document start of a stream"""

    def __init__(self, impl=""):
        L = C.CDLL(REF_GRAM_SO)
        L.sjr_grammar_supported.restype = C.c_int
        L.sjr_grammar_supported.argtypes = [C.c_char_p]
        L.sjr_parse_error.restype = C.c_int
        L.sjr_parse_error.argtypes = [C.c_char_p, C.POINTER(C.c_uint8), C.c_size_t, C.c_size_t]
        L.sjr_stream_errors.restype = C.c_int
        L.sjr_stream_errors.argtypes = [C.c_char_p, C.POINTER(C.c_uint8), C.c_size_t, C.c_int, C.c_size_t, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_int),
                                        C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        self.L = L
        self.impl = impl.encode()
        if not L.sjr_grammar_supported(self.impl):
            raise RuntimeError(f"reference implementation {impl!r} not supported on this host")

    def parse(self, buf, max_depth=1024):
        a = np.frombuffer(bytes(buf) + b"\0", dtype=np.uint8)
        return self.L.sjr_parse_error(self.impl, _ptr(a), len(buf), max_depth)

    def stream(self, buf, starts, max_depth=1024, mode=O.REGULAR):
        """stage2_next from each start: (stage-1 error, error per start, next_structural_index per start (NONE on an
        error), n); mode REGULAR keeps incomplete last documents, which STREAMING_FINAL drops"""
        a = np.frombuffer(bytes(buf) + b"\0", dtype=np.uint8)
        D = max(len(starts), 1)
        st = (C.c_uint32 * D)(*starts)
        errs = (C.c_int * D)()
        nxt = (C.c_uint32 * D)()
        n = C.c_uint32(0)
        e = self.L.sjr_stream_errors(self.impl, _ptr(a), len(buf), mode, max_depth, st, len(starts), errs, nxt, C.byref(n))
        return e, list(errs)[: len(starts)], list(nxt)[: len(starts)], n.value


# ---- cases
LEAVES = [b'"s"', b'1', b'-2', b'3.5', b'1e2', b'true', b'false', b'null', b'{}', b'[]', b'18446744073709551615']
BAD_LEAVES = [b'"\\x"', b'01', b'-', b'1.', b'tru', b'fals', b'nul', b'99999999999999999999999', b'+1', b'#', b'x']


def grammar_cases():
    """every return of walk_document (L120-244), every token error as root / key / value, around grammar errors"""
    c = [
        # TAPE_ERROR of the walk
        b'[1 2]', b'{"a" 1}', b'[1,]', b'{"a":1]', b'[1]]', b'{"a":1,}', b'{1:2}', b'{"a":1 "b":2}', b'{,}', b'[,1]', b'[1,,2]', b'{"a"}',
        b'{"a":}', b'{:1}', b'[}', b'{]', b'[:]', b'{"a"::1}', b'["a":1]', b'[1:2]', b'{"a",1}', b'1 2', b'[] []', b'{} 1', b'"a" "b"',
        b'[1]x', b']', b'}', b',', b':', b'[', b'{', b'[[]', b'[{}', b'[[1],', b'{"a":[1,{"b":2]}', b'{"a":{"b":[}}}',
        # the unmatched root bracket
        b'[1,2', b'{"a":1', b'[1]  ,', b'{"a":1} ]', b'[{"a":1}', b'[] 1', b'{}]',
        # empty containers
        b'{}', b'[]', b'[{}]', b'{"a":[]}', b'[[],[[]],{}]', b'{"a":{},"b":[]}',
        b'', b'   ',
    ]
    for leaf in LEAVES + BAD_LEAVES:
        c += [leaf, b'[' + leaf + b']', b'{"k":' + leaf + b'}', b'{' + leaf + b':1}', b'[1,' + leaf + b',2]', b'{"a":1,' + leaf + b':2}',
              b'[' + leaf + b' 1]', b'[1 ' + leaf + b']', b'{"a":' + leaf + b' "b":1}', b'[' + leaf + b',]']
    return c


def nested(depth, inner=b"1", kind="["):
    o, c = (b"[", b"]") if kind == "[" else (b'{"k":', b"}")
    return o * depth + inner + c * depth


def depth_cases():
    """(document, max_depth) around the depth limit, with empty containers at the limit"""
    out = []
    for md in (1, 2, 3, 1024, 4096):
        for d in sorted({max(md - 2, 0), max(md - 1, 0), md, md + 1}):
            for inner in (b"1", b"[]", b"{}", b'[1]'):
                out.append((nested(d, inner), md))
                out.append((nested(d, inner, "{"), md))
    return out


def stream_cases():
    """streams where documents meet: root scalars at the buffer's end and glued to the next document"""
    return [b'1"a"', b'true"x"', b'1 2 3', b'[1] 2 {"a":3}', b'"x"[1]', b'nul 1', b'[1]{"a":2}3', b'1[', b'[1] [2', b'{"a":1}{"b"',
            b'1 tru', b'[1 tru] 2', b'[1,2] [3 4] [5]', b'{"a":1} [2,] 3', b'1', b'true', b'"abc"', b'-0', b'[]{}', b'{}{}[][]']


def mutate_once(doc, rng, port):
    """delete, duplicate or swap structurals of doc: the token at a structural runs up to the next one"""
    r = port.stage1(doc)
    idx = [int(i) for i in r.idx[: r.n]] if r.err == 0 else []
    if len(idx) < 2:
        return doc
    span = lambda k: (idx[k], idx[k + 1] if k + 1 < len(idx) else len(doc))  # noqa: E731
    s, e = span(rng.randrange(len(idx)))
    op = rng.choice(("del", "dup", "swap"))
    if op == "del":
        return doc[:s] + doc[e:]
    if op == "dup":
        return doc[:s] + doc[s:e] + doc[s:]
    a, b = sorted([(s, e), span(rng.randrange(len(idx)))])
    if a == b or a[1] > b[0]:
        return doc
    return doc[: a[0]] + doc[b[0]:b[1]] + doc[a[1]:b[0]] + doc[a[0]:a[1]] + doc[b[1]:]


def fuzz_docs(count, seed=7):
    """seeded mutations (one or two) of random documents and of twitter / amazon rows, kept when stage 1 still passes"""
    import pointer_cases as PC
    rng = random.Random(seed)
    port = O.Port()
    base = PC.random_docs(12, seed) + PC.twitter_rows()[:20] + PC.amazon_rows(40)[:20]
    out = []
    while len(out) < count:
        m = rng.choice(base)
        if rng.random() < 0.9:
            for _ in range(rng.choice((1, 2))):
                m = mutate_once(m, rng, port)
        if port.stage1(m).err == 0:
            out.append(m)
    return out


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)


# ---- what the reference's answers mean for ours
def expected_from_ref(err, next_index, starts, d, n):
    """the (error, index) the reference's stage2_next implies for document d of a table: SUCCESS that stops before the
    document's end is our TAPE_ERROR at the first structural left over; an error's index is not exposed (None)"""
    end = starts[d + 1] if d + 1 < len(starts) else n
    if err:
        return err, None
    return (0, end) if next_index == end else (TAPE_ERROR, next_index)


def agrees(doc, r, starts, d, err, idx, want_err, want_idx):
    """our verdict against the reference's, with the documented deviations: a root token that starts with a byte below
    '0' other than '-' (NUMBER_ERROR here, TAPE_ERROR there), a float whose value is infinite (SUCCESS here,
    NUMBER_ERROR there) and the last document of a stream wanting a value past n, where the reference reads its zero
    padding (a NUMBER_ERROR there) and ours is a TAPE_ERROR at n"""
    if err == want_err and (want_idx is None or idx == want_idx):
        return True
    if err == NUMBER_ERROR and want_err == TAPE_ERROR and r.n and idx == (starts[d] if starts else 0):
        b = doc[r.idx[starts[d] if starts else 0]]
        return b < ord("0") and b != ord("-")
    if err == TAPE_ERROR and idx == r.n and starts and want_err in (NUMBER_ERROR, TAPE_ERROR):
        return d == len(starts) - 1
    return False
