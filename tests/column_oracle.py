"""ctypes bindings for the two typed-column checkers (test infrastructure only; recipe: oracle/column.mk).

  Columns    : oracle/libsj_column_oracle.so    -- sjo_column, our C restatement of the DOM getters on one JSON
                                                  Pointer result over the oracle's tokens (always built)
  RefColumns : oracle/_ref/libsj_ref_column.so  -- the unmodified reference's at_pointer + getter (may be absent)
"""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O
import pointer_oracle as PO

ORACLE_DIR = O.ORACLE_DIR
MAKEFILE = os.path.join(ORACLE_DIR, "column.mk")
COL_SO = os.path.join(ORACLE_DIR, "libsj_column_oracle.so")
REF_COL_SO = os.path.join(ORACLE_DIR, "_ref", "libsj_ref_column.so")

INT64, UINT64, BOOL, STRING, ARRAY_SIZE, OBJECT_SIZE = 1, 2, 3, 4, 5, 6
KINDS = (INT64, UINT64, BOOL, STRING, ARRAY_SIZE, OBJECT_SIZE)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Columns:
    """sjo_column over tokens (Port.tokens() output) and rows {error, index}"""

    def __init__(self):
        if not os.path.exists(COL_SO) or os.path.getmtime(COL_SO) < os.path.getmtime(os.path.join(ORACLE_DIR, "sj_column_oracle.c")):
            subprocess.check_call(["make", "-f", MAKEFILE, COL_SO], stdout=subprocess.DEVNULL)
        L = C.CDLL(COL_SO)
        L.sjo_column.restype = C.c_int
        L.sjo_column.argtypes = [C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.c_uint32, C.POINTER(C.c_uint8), C.c_size_t, C.c_int32, C.c_uint32,
                                 C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        self.L = L

    def column(self, kind, types, payload, strbuf, string_bytes, rows_err, rows_idx):
        """(error int32[R], row_type uint8[R], values uint64[R], strings [bytes]) of every row"""
        n = len(types)
        t = np.ascontiguousarray(types, dtype=np.uint8) if n else np.zeros(1, dtype=np.uint8)
        pl = np.ascontiguousarray(payload, dtype=np.uint64) if n else np.zeros(1, dtype=np.uint64)
        sb = np.ascontiguousarray(strbuf, dtype=np.uint8) if len(strbuf) else np.zeros(1, dtype=np.uint8)
        re_ = np.asarray(rows_err, dtype=np.int64).ravel()
        ri = np.asarray(rows_idx, dtype=np.int64).ravel() & 0xFFFFFFFF
        R = len(re_)
        err = np.zeros(R, dtype=np.int32)
        rt = np.zeros(R, dtype=np.uint8)
        val = np.zeros(R, dtype=np.uint64)
        strs = []
        ty, v, so, sl = C.c_uint8(), C.c_uint64(), C.c_uint64(), C.c_uint32()
        tp, pp, sp = _p(t, C.c_uint8), _p(pl, C.c_uint64), _p(sb, C.c_uint8)
        for r in range(R):
            err[r] = self.L.sjo_column(kind, tp, pp, n, sp, string_bytes, int(re_[r]), int(ri[r]), C.byref(ty), C.byref(v), C.byref(so), C.byref(sl))
            rt[r], val[r] = ty.value, v.value
            if kind == STRING:
                strs.append(bytes(sb[so.value: so.value + sl.value]) if sl.value else b"")
        return err, rt, val, strs

    def of_document(self, kind, doc, pointers, starts=None):
        """stage 1, tokens and at_pointer of the pointer oracle, then the column of every (pointer, document):
        (pointer table (stage1, tokens, starts, err, idx), error[P, D], row_type[P, D], values[P, D], strings)"""
        tab = PO.Pointers().table(doc, pointers, starts=starts)
        _r, tw, _s, perr, pidx = tab
        err, rt, val, strs = self.column(kind, tw[1], tw[2], tw[3], len(tw[3]), perr, pidx)
        shape = perr.shape
        return tab, err.reshape(shape), rt.reshape(shape), val.reshape(shape), strs


def have_ref():
    return os.path.exists(REF_COL_SO)


class RefColumns:
    """the unmodified reference: dom::parser::parse once, then at_pointer and the getter of each pointer"""

    def __init__(self):
        L = C.CDLL(REF_COL_SO)
        L.sjr_dom_column.restype = C.c_int
        L.sjr_dom_column.argtypes = [C.POINTER(C.c_uint8), C.c_size_t, C.c_char_p, C.POINTER(C.c_size_t), C.c_int, C.c_int, C.POINTER(C.c_int),
                                     C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        self.L = L

    def column(self, kind, buf, pointers):
        """(parse error, [(error, value, bytes)] per pointer)"""
        a = np.frombuffer(bytes(buf), dtype=np.uint8) if len(buf) else np.zeros(1, dtype=np.uint8)
        ps = [p.encode() if isinstance(p, str) else bytes(p) for p in pointers]
        k = max(len(ps), 1)
        lens = (C.c_size_t * k)(*[len(p) for p in ps])
        errs = (C.c_int * k)()
        vals = (C.c_uint64 * k)()
        olens = (C.c_size_t * k)()
        cap = len(buf) + 64
        for _ in range(2):
            out = C.create_string_buffer(cap)
            perr = self.L.sjr_dom_column(_p(a, C.c_uint8), len(buf), b"".join(ps), lens, len(ps), kind, errs, vals, out, cap, olens)
            if sum(olens[: len(ps)]) <= cap:
                break
            cap = sum(olens[: len(ps)])
        res, at = [], 0
        for i in range(len(ps)):
            res.append((errs[i], vals[i], out.raw[at: at + olens[i]]))
            at += olens[i]
        return perr, res
