"""Shared by test_stream_fold.py (CPU) and test_sharded_streams.py (GPU): inputs and cuts for sharded stream passes, the
oracle's view of every shard, and the check of a pass's per-rank results against stage1(whole buffer, mode).

Gathering rule: G = concat over ranks of d_idx[0:count] + bytes_before, followed by the last rank's three words after its
count (the first two + its bytes_before, the third as is); G[0:n+3] must equal the whole call's words (uint32 arithmetic)."""
import ctypes as C

import numpy as np

import oracle_lib as O
from simdjson_b200 import corpus

ROLE = {ord(":"): 1, ord(","): 1, ord("{"): 2, ord("}"): 3, ord("["): 4, ord("]"): 5}


def role(c):
    return ROLE.get(int(c), 0)


def starts(cur, before):
    if cur in (1, 3, 5):
        return False
    return before not in (2, 4, 1)


def doc_starts(buf, idx, n):
    """every i < n where a document starts (structural 0 always), as sjb200_document_table_dev defines it"""
    return [i for i in range(n) if i == 0 or starts(role(buf[idx[i]]), role(buf[idx[i - 1]]))]


def inputs(rng):
    """(name, bytes) of the streams the sharded tests cut"""
    out = [(f"multi{i}", corpus.multi_document(rng)) for i in range(40)]
    out += [(f"adv{i}", corpus.adversarial(rng)) for i in range(40)]
    rows = bytes(corpus.ndjson_rows(24000))
    out.append(("ndjson_cut", rows[: len(rows) - 157]))  # the last row cut short
    out.append(("ndjson", rows))
    out.append(("mixed", b'[1,2,3]  {"a":1} [1,2  '))
    out.append(("string_ranks_before_end", b'{"a":1} [2] {"b":"x"} "' + b"abc def " * 400))  # ends inside a string
    out.append(("whitespace_run", b'{"a":[1,2]}' + b" " * 300 + b"\n" * 100 + b'["x"] 7'))
    out.append(("partial_utf8_tail", b'{"u":"\xc3\xa9"} [1] {"v":2}\xe2\x82'))
    out.append(("pretty", b'{\n  "a": [\n    1,\n    {"b": "c \\" d"}\n  ],\n  "e": {"f": null}\n}\n'))
    return out


def _boundary(buf, pos):
    while 0 < pos < len(buf) and (buf[pos] & 0xC0) == 0x80:
        pos -= 1
    return pos


def cut_sets(rng, buf, world, count):
    """up to `count` sets of world-1 cuts at character boundaries (every shard >= 1 byte).  Candidates: random bytes,
    right after an opening bracket, inside whitespace runs, and the start of a partial UTF-8 character at the end"""
    n = len(buf)
    if n < world:
        return []
    special = [i + 1 for i, c in enumerate(buf) if c in (ord("{"), ord("[")) and i + 1 < n]
    special += [i for i in range(1, n) if buf[i] in (0x20, 0x0A) and buf[i - 1] in (0x20, 0x0A)]
    special += [i for i in range(max(1, n - 3), n) if buf[i] >= 0xC0]
    sets = []
    for _ in range(count * 4):
        if len(sets) >= count:
            break
        picks = set()
        while len(picks) < world - 1:
            p = rng.choice(special) if special and rng.random() < 0.5 else rng.randrange(1, n)
            picks.add(p)
        cuts = [0] + sorted(_boundary(buf, p) for p in picks) + [n]
        if all(cuts[k + 1] > cuts[k] for k in range(world)) and cuts not in sets:
            sets.append(cuts)
    return sets


class Oracle:
    def __init__(self):
        self.port = O.Port()
        L = self.port.L
        L.sjo_scan_shard.restype = C.c_uint64
        L.sjo_scan_shard.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]

    def scan(self, shard, state_in):
        """(structurals, shard-relative indexes, state out) of a shard entered in state_in"""
        a = np.frombuffer(bytes(shard), dtype=np.uint8)
        idx = np.zeros(len(a) + 4, dtype=np.uint32)
        so = C.c_uint32(0)
        k = self.port.L.sjo_scan_shard(a.ctypes.data if len(a) else None, len(a), state_in, idx.ctypes.data, C.byref(so))
        return int(k), idx[: int(k)], int(so.value)

    def trim(self, shard):
        a = np.frombuffer(bytes(shard), dtype=np.uint8)
        return int(self.port.L.sjo_trim_partial_utf8(a.ctypes.data_as(C.POINTER(C.c_uint8)), len(a))) if len(a) else 0

    def shards(self, buf, cuts, mode):
        """the shards as a pass sees them (last one trimmed in the streaming modes), or None when that trim differs from
        the whole buffer's (only possible for invalid UTF-8 right before the last cut)"""
        sh = [bytes(buf[cuts[r]: cuts[r + 1]]) for r in range(len(cuts) - 1)]
        if mode != O.REGULAR:
            t = self.trim(sh[-1])
            if cuts[-2] + t != self.trim(buf):
                return None
            sh[-1] = sh[-1][:t]
        return sh

    def summaries(self, buf, cuts, mode):
        """what every rank's scan and summary kernel produce: (summaries, final_state, flags_all, per-rank indexes)"""
        sh = self.shards(buf, cuts, mode)
        if sh is None:
            return None
        state, scans = 0, []
        for s in sh:
            k, idx, state = self.scan(s, state)
            scans.append((k, idx))
        whole = b"".join(sh)
        unclosed = bool(state & 2)
        flags = 0 if self.port.validate_utf8(whole) else 1
        if self.port.stage1(whole, O.STREAMING_FINAL).err == O.UNESCAPED_CHARS:
            flags |= 2
        holder = max([r for r, (k, _) in enumerate(scans) if k] or [-1])
        sums = []
        for r, (s, (k, idx)) in enumerate(zip(sh, scans)):
            kp = k - (1 if mode != O.REGULAR and unclosed and r == holder else 0)
            roles = [role(s[i]) for i in idx[:kp]]
            start, nobj, narr = -1, 0, 0
            if mode != O.REGULAR and kp:
                for i in range(kp - 1, 0, -1):
                    if starts(roles[i], roles[i - 1]):
                        start = i
                        break
                for x in roles[max(start, 0):]:
                    nobj += (x == 2) - (x == 3)
                    narr += (x == 4) - (x == 5)
            sums.append(dict(count=k, len=len(s), first_byte=int(idx[0]) if k else 0, last_byte=int(idx[k - 1]) if k else 0,
                             start_index=max(start, 0), start_byte=int(idx[start]) if start >= 0 else 0, net_obj=nobj, net_arr=narr,
                             role_first=roles[0] if kp else 0, role_last=roles[-1] if kp else 0, has_start=int(start >= 0)))
        return sums, state, flags, [idx for _, idx in scans]


def check(buf, cuts, mode, want, ranks):
    """ranks[r] = dict(err, n, kept, bytes_before, total_bytes, first_starts_document, count, words): words = the rank's
    d_idx[0:count] (+ 3 more words on the last rank) after the pass.  want = port.stage1(whole buffer, mode)."""
    world = len(ranks)
    tag = (len(buf), cuts, mode)
    for r, g in enumerate(ranks):
        assert g["err"] == want.err, (tag, r, g["err"], want.err)
        assert g["bytes_before"] == cuts[r], (tag, r)
    if not want.wrote:
        for r, g in enumerate(ranks):
            assert g["n"] == 0 and g["kept"] == 0, (tag, r)
        return
    n = want.n
    base = 0
    parts = []
    for r, g in enumerate(ranks):
        assert g["n"] == n, (tag, r, g["n"], n)
        assert g["kept"] == min(max(n - base, 0), g["count"]), (tag, r, g["kept"])
        w = np.asarray(g["words"], dtype=np.uint32)
        off = np.uint32(g["bytes_before"] & 0xFFFFFFFF)
        if r < world - 1:
            parts.append(w[: g["count"]] + off)
        else:
            parts.append(w[: g["count"] + 2] + off)
            parts.append(w[g["count"] + 2: g["count"] + 3])
        base += g["count"]
    G = np.concatenate(parts)
    assert np.array_equal(G[: n + 3], want.idx[: n + 3]), (tag, G[: n + 3][-6:], want.idx[: n + 3][-6:])
    if mode == O.STREAMING_FINAL:
        assert all(g["total_bytes"] == int(want.idx[n]) for g in ranks), tag
    # first_starts_document: is the rank's first kept structural a document start of the whole stream's first n?
    starts_all = set(doc_starts(np.frombuffer(bytes(buf), dtype=np.uint8), want.idx, n))
    base = 0
    for r, g in enumerate(ranks):
        if g["kept"]:
            assert bool(g["first_starts_document"]) == (base in starts_all), (tag, r)
        base += g["count"]

