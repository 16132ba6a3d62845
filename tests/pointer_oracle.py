"""ctypes bindings for the two JSON Pointer checkers (test infrastructure only; recipe: oracle/pointer.mk).

  Pointers    : oracle/libsj_pointer_oracle.so      -- sjo_at_pointer, our recursive C restatement of
                                                       dom::element::at_pointer over the oracle's tokens (always built)
  RefPointers : oracle/_ref/libsj_ref_pointer.so    -- the unmodified reference's at_pointer (may be absent)

plus document_starts / value_span, the stream and span helpers the pointer tests share.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O

ORACLE_DIR = O.ORACLE_DIR
MAKEFILE = os.path.join(ORACLE_DIR, "pointer.mk")
PTR_SO = os.path.join(ORACLE_DIR, "libsj_pointer_oracle.so")
REF_PTR_SO = os.path.join(ORACLE_DIR, "_ref", "libsj_ref_pointer.so")


def _u8(buf):
    if isinstance(buf, (bytes, bytearray)):
        return np.frombuffer(bytes(buf), dtype=np.uint8)
    return np.ascontiguousarray(buf, dtype=np.uint8)


def _ptr(a, t=C.c_uint8):
    return a.ctypes.data_as(C.POINTER(t))


def _enc(p):
    return p.encode() if isinstance(p, str) else bytes(p)


class Pointers:
    """sjo_at_pointer over the tokens of oracle_lib.Port (stage 1 and stage-2-lite of the pinned C restatement)"""

    def __init__(self):
        if not os.path.exists(PTR_SO) or os.path.getmtime(PTR_SO) < os.path.getmtime(os.path.join(ORACLE_DIR, "sj_pointer_oracle.c")):
            subprocess.check_call(["make", "-f", MAKEFILE, PTR_SO], stdout=subprocess.DEVNULL)
        L = C.CDLL(PTR_SO)
        L.sjo_at_pointer.restype = C.c_int
        L.sjo_at_pointer.argtypes = [C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.c_uint32, C.POINTER(C.c_uint8), C.c_size_t, C.c_uint32, C.c_uint32,
                                     C.c_char_p, C.c_size_t, C.POINTER(C.c_uint32)]
        self.L = L
        self.port = O.Port()

    def at_pointer(self, types, payload, strbuf, pointer, root=0, end=None):
        """dom::element::at_pointer of the document at structurals [root, end) of Port.tokens() output: (error, index)"""
        n = len(types)
        t = np.ascontiguousarray(types, dtype=np.uint8) if n else np.zeros(1, dtype=np.uint8)
        pl = np.ascontiguousarray(payload, dtype=np.uint64) if n else np.zeros(1, dtype=np.uint64)
        sb = np.ascontiguousarray(strbuf, dtype=np.uint8) if len(strbuf) else np.zeros(1, dtype=np.uint8)
        p = _enc(pointer)
        ix = C.c_uint32(0)
        err = self.L.sjo_at_pointer(_ptr(t), _ptr(pl, C.c_uint64), n, _ptr(sb), len(strbuf), root, n if end is None else end, p, len(p), C.byref(ix))
        return err, ix.value

    def table(self, buf, pointers, mode=O.REGULAR, starts=None):
        """stage 1, tokens and at_pointer of every pointer in every document: (stage1 result, tokens result, document starts,
        error int32[P, D], index uint32[P, D]); starts defaults to one document at structural 0"""
        r = self.port.stage1(buf, mode)
        tw = self.port.tokens(buf, r.idx, r.n)
        starts = [0] if starts is None else list(starts)
        err = np.zeros((len(pointers), len(starts)), dtype=np.int32)
        idx = np.zeros((len(pointers), len(starts)), dtype=np.uint32)
        for d, s in enumerate(starts):
            end = starts[d + 1] if d + 1 < len(starts) and starts[d + 1] > s else r.n
            for p, ptr in enumerate(pointers):
                err[p, d], idx[p, d] = self.at_pointer(tw[1], tw[2], tw[3], ptr, s, end)
        return r, tw, starts, err, idx


def have_ref():
    return os.path.exists(REF_PTR_SO) and O.have_ref()


class RefPointers:
    """the unmodified reference: dom::parser::parse once, then at_pointer of each pointer"""

    def __init__(self, impl=""):
        L = C.CDLL(REF_PTR_SO)
        L.sjr_pointer_supported.restype = C.c_int
        L.sjr_pointer_supported.argtypes = [C.c_char_p]
        L.sjr_dom_at_pointer.restype = C.c_int
        L.sjr_dom_at_pointer.argtypes = [C.c_char_p, C.POINTER(C.c_uint8), C.c_size_t, C.c_char_p, C.POINTER(C.c_size_t), C.c_int, C.POINTER(C.c_int), C.c_char_p,
                                         C.c_size_t, C.POINTER(C.c_size_t)]
        self.L = L
        self.impl = impl.encode()
        if not L.sjr_pointer_supported(self.impl):
            raise RuntimeError(f"reference implementation {impl!r} not supported on this host")

    def at_pointer(self, buf, pointers):
        """[(error_code, minified element)] per pointer"""
        a = _u8(buf)
        ps = [_enc(p) for p in pointers]
        k = max(len(ps), 1)
        lens = (C.c_size_t * k)(*[len(p) for p in ps])
        errs = (C.c_int * k)()
        olens = (C.c_size_t * k)()
        cap = 16 * len(a) + (1 << 20)
        for _ in range(2):  # the second time with room for everything the first one counted
            out = C.create_string_buffer(cap)
            self.L.sjr_dom_at_pointer(self.impl, _ptr(a), len(a), b"".join(ps), lens, len(ps), errs, out, cap, olens)
            if sum(olens[: len(ps)]) <= cap:
                break
            cap = sum(olens[: len(ps)])
        res, at = [], 0
        for i in range(len(ps)):
            res.append((errs[i], out.raw[at: at + olens[i]]))
            at += olens[i]
        return res


def document_starts(buf, idx, n):
    """structural indexes at which the documents of a whitespace-separated stream start: the predicate of
    find_next_document_index at every position (what sjb200_document_table_dev computes)"""
    a = _u8(buf)
    starts = [0] if n else []
    for i in range(1, n):
        c, prev = a[idx[i]], a[idx[i - 1]]
        if c not in b"}],:" and prev not in b"{[,:":
            starts.append(i)
    return starts


def value_span(buf, idx, types, k):
    """the raw bytes of the value at structural k: from idx[k] to the end of that value"""
    a = bytes(_u8(buf))
    if types[k] in (ord("{"), ord("[")):
        depth = 0
        for j in range(k, len(types)):
            if types[j] in (ord("{"), ord("[")):
                depth += 1
            elif types[j] in (ord("}"), ord("]")):
                depth -= 1
                if depth == 0:
                    return a[idx[k]: idx[j] + 1]
        return a[idx[k]:]
    end = idx[k + 1] if k + 1 < len(types) else len(a)
    return a[idx[k]: end].rstrip(b" \t\r\n")
