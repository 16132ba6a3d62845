"""ctypes bindings for the two get_double checkers (test infrastructure only; recipe: oracle/double.mk).

  Doubles    : oracle/libsj_double_oracle.so    -- sjo_double, our C restatement of element::get_double on one JSON
                                                  Pointer result over the oracle's tokens (always built)
  RefDoubles : oracle/_ref/libsj_ref_double.so  -- the unmodified reference's parse + at_pointer + get_double (may be absent)
"""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O

ORACLE_DIR = O.ORACLE_DIR
MAKEFILE = os.path.join(ORACLE_DIR, "double.mk")
DBL_SO = os.path.join(ORACLE_DIR, "libsj_double_oracle.so")
REF_DBL_SO = os.path.join(ORACLE_DIR, "_ref", "libsj_ref_double.so")


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Doubles:
    """sjo_double over the input, its structurals, tokens (Port.tokens() output) and rows {error, index}"""

    def __init__(self):
        if not os.path.exists(DBL_SO) or os.path.getmtime(DBL_SO) < os.path.getmtime(os.path.join(ORACLE_DIR, "sj_double_oracle.c")):
            subprocess.check_call(["make", "-f", MAKEFILE, DBL_SO], stdout=subprocess.DEVNULL)
        L = C.CDLL(DBL_SO)
        L.sjo_double.restype = C.c_int
        L.sjo_double.argtypes = [C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.c_uint32, C.POINTER(C.c_uint8), C.c_size_t, C.POINTER(C.c_uint32),
                                 C.c_int32, C.c_uint32, C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)]
        self.L = L

    def column(self, buf, idx, types, payload, rows_err, rows_idx, length=None):
        """(error int32[R], row_type uint8[R], bits uint64[R]) of every row; length: the input's length (default len(buf))"""
        n = len(types)
        b = np.frombuffer(bytes(buf), dtype=np.uint8) if len(buf) else np.zeros(1, dtype=np.uint8)
        ix = np.ascontiguousarray(idx, dtype=np.uint32) if len(idx) else np.zeros(1, dtype=np.uint32)
        t = np.ascontiguousarray(types, dtype=np.uint8) if n else np.zeros(1, dtype=np.uint8)
        pl = np.ascontiguousarray(payload, dtype=np.uint64) if n else np.zeros(1, dtype=np.uint64)
        re_ = np.asarray(rows_err, dtype=np.int64).ravel()
        ri = np.asarray(rows_idx, dtype=np.int64).ravel() & 0xFFFFFFFF
        R = len(re_)
        err = np.zeros(R, dtype=np.int32)
        rt = np.zeros(R, dtype=np.uint8)
        val = np.zeros(R, dtype=np.uint64)
        ty, v = C.c_uint8(), C.c_uint64()
        bp, ip, tp, pp = _p(b, C.c_uint8), _p(ix, C.c_uint32), _p(t, C.c_uint8), _p(pl, C.c_uint64)
        ln = len(buf) if length is None else length
        for r in range(R):
            err[r] = self.L.sjo_double(tp, pp, n, bp, ln, ip, int(re_[r]), int(ri[r]), C.byref(ty), C.byref(v))
            rt[r], val[r] = ty.value, v.value
        return err, rt, val

    def of_text(self, text):
        """(error, row_type, bits) of get_double on the one element of the document [text]"""
        doc = b"[" + text.encode() + b"]"
        port = O.Port()
        r = port.stage1(doc)
        tw = port.tokens(doc, r.idx, r.n)
        e, t, v = self.column(doc, r.idx[: r.n], tw[1], tw[2], [0], [1])
        return int(e[0]), int(t[0]), int(v[0])


def have_ref():
    return os.path.exists(REF_DBL_SO)


class RefDoubles:
    """the unmodified reference: dom::parser::parse once, then at_pointer and get_double of each pointer"""

    def __init__(self):
        L = C.CDLL(REF_DBL_SO)
        L.sjr_dom_double.restype = C.c_int
        L.sjr_dom_double.argtypes = [C.POINTER(C.c_uint8), C.c_size_t, C.c_char_p, C.POINTER(C.c_size_t), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
        self.L = L

    def column(self, buf, pointers):
        """(parse error, [(error, bits)] per pointer)"""
        a = np.frombuffer(bytes(buf), dtype=np.uint8) if len(buf) else np.zeros(1, dtype=np.uint8)
        ps = [p.encode() if isinstance(p, str) else bytes(p) for p in pointers]
        k = max(len(ps), 1)
        lens = (C.c_size_t * k)(*[len(p) for p in ps])
        errs = (C.c_int * k)()
        vals = (C.c_uint64 * k)()
        perr = self.L.sjr_dom_double(_p(a, C.c_uint8), len(buf), b"".join(ps), lens, len(ps), errs, vals)
        return perr, [(errs[i], vals[i]) for i in range(len(ps))]

    def of_text(self, text):
        """(error, bits) of get_double on the one element of the document [text]"""
        _perr, res = self.column(b"[" + text.encode() + b"]", ["/0"])
        return res[0]
