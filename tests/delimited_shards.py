"""Shared by test_delimited_fold.py (CPU) and test_sharded_delimited.py (GPU): inputs and cuts for sharded RS-delimited
and comma-delimited passes (modes 3-6), a Python model of what every rank's carry and filter rounds produce (the device
filter of sjb200_docs.cu with the carried-in depth / run), and the check of a pass's per-rank results against
stage1(whole buffer, mode).

Gathering rule: G = concat over ranks of (d_idx[0:kept] + bytes_before) (mod 2^32), followed by tail[0..2]; G[0:n+3]
must equal the whole call's words."""
import random

import numpy as np

import oracle_lib as O
import stream_shards as S
from simdjson_b200 import corpus

RS = 0x1E
WS = (0x20, 0x09, 0x0A, 0x0D)
MODES = (O.JSON_SEQUENCE_PARTIAL, O.JSON_SEQUENCE_FINAL, O.COMMA_DELIMITED_PARTIAL, O.COMMA_DELIMITED_FINAL)


def is_rs_mode(mode):
    return mode in (O.JSON_SEQUENCE_PARTIAL, O.JSON_SEQUENCE_FINAL)


def _ws_rs(c):
    return c in WS or c == RS


# the cases DESIGN.md section 5 names, as RS streams (rs) and comma streams (comma)
def special_inputs():
    rs = [
        ("rs_run_spanning", b"\x1e{\"a\":1}\n\x1e  \x1e \n\x1e" + b" " * 200 + b"\x1e\n\x1e  [1,2]\n\x1e" + b" \n" * 150 + b"\x1e7\n"),
        ("rs_glued_scalar", b"\x1e123\x1e456\x1e \x1e\"s\"\x1e  true\x1e\x1enull"),
        ("rs_glued_behind_scalar", b"\x1e1\x1e \x1e2 \x1e{\"x\":1\x1e}\x1e3\x1e"),
        ("rs_one_sep", b"\x1e{\"a\":[1,2,3]}"),
        ("rs_no_sep", b"{\"a\":1} [2]"),
        ("rs_string_tail", b"\x1e{\"a\":1}\n\x1e\"" + b"abc \x1e def " * 40),
        ("rs_partial_utf8", b"\x1e{\"u\":\"\xc3\xa9\"}\n\x1e[1]\n\x1e\xe2\x82"),
        ("rs_ws_only_tail", b"\x1e[1]\n\x1e" + b"  \n" * 100),
    ]
    comma = [
        ("comma_negative_depth", b"[1,[2]],{}]],{},3,[4,{\"a\":[5,6]}],7"),
        ("comma_no_root", b"[1,2,3,{\"a\":[4,5]}]"),
        ("comma_string_tail", b"{\"a\":1},[2],\"" + b"x, y, " * 60),
        ("comma_partial_utf8", b"{\"a\":\"\xc3\xa9\"},[1],2\xf0\x9f\x98"),
        ("comma_scalars", b"1,2,3,\"a,b\",true,null,[7,8],{\"k\":9}"),
        ("comma_spaces", b"1 , 2 ,\n[3 , 4] , " + b" " * 300 + b"{ \"z\" : 5 }"),
    ]
    return rs, comma


def inputs(rng, nfuzz=40):
    """(name, bytes, modes) of the streams the delimited tests cut: the fuzz RS / comma streams of the single-GPU parity
    test, NDJSON rows as RS and comma streams, and the special cases"""
    rs_modes, comma_modes = MODES[:2], MODES[2:]
    out = []
    for i in range(nfuzz):
        out.append((f"rsfuzz{i}", b"\x1e" + corpus.multi_document(rng, sep=b"\x1e"), rs_modes))
        out.append((f"commafuzz{i}", corpus.multi_document(rng, sep=b","), comma_modes))
    rows = bytes(corpus.ndjson_rows(6000)).split(b"\n")
    rows = [r for r in rows if r]
    out.append(("rs_rows", b"".join(b"\x1e" + r + b"\n" for r in rows), rs_modes))
    out.append(("comma_rows", b",".join(rows), comma_modes))
    out.append(("comma_rows_cut", b",".join(rows)[:-37], comma_modes))
    rs, comma = special_inputs()
    out += [(n, b, rs_modes) for n, b in rs] + [(n, b, comma_modes) for n, b in comma]
    return out


def _boundary(buf, pos):
    while 0 < pos < len(buf) and (buf[pos] & 0xC0) == 0x80:
        pos -= 1
    return pos


def cut_sets(rng, buf, world, count):
    """up to `count` sets of world-1 cuts at character boundaries: random bytes, right after an RS, inside RS /
    whitespace runs, right before a scalar glued to an RS, right after a root comma, inside strings"""
    n = len(buf)
    if n < world:
        return []
    special = [i + 1 for i, c in enumerate(buf) if c == RS and i + 1 < n]
    special += [i for i in range(1, n) if _ws_rs(buf[i]) and _ws_rs(buf[i - 1])]
    special += [i for i in range(1, n) if buf[i - 1] == RS and not _ws_rs(buf[i])]
    special += [i + 1 for i, c in enumerate(buf) if c == ord(",") and i + 1 < n]
    special += [i + 1 for i, c in enumerate(buf) if c == ord('"') and i + 1 < n]
    special += [i for i in range(max(1, n - 3), n) if buf[i] >= 0xC0]
    sets = []
    for _ in range(count * 4):
        if len(sets) >= count:
            break
        picks = set()
        while len(picks) < world - 1:
            p = rng.choice(special) if special and rng.random() < 0.6 else rng.randrange(1, n)
            picks.add(p)
        cuts = [0] + sorted(_boundary(buf, p) for p in picks) + [n]
        if all(cuts[k + 1] > cuts[k] for k in range(world)) and cuts not in sets:
            sets.append(cuts)
    return sets


# ------------------------------------------------------------------------------------------------- the model
def carry(shard, idx, n, comma):
    """the carry round's words of one shard (n: the structurals its filter considers)"""
    if comma:
        net = 0
        for i in idx[:n]:
            r = S.role(shard[i])
            net += (r in (2, 4)) - (r in (3, 5))
        return dict(len=len(shard), net=net)
    lo = int(idx[n - 1]) + 1 if n else 0
    ok = all(_ws_rs(c) for c in shard[lo:])
    return dict(len=len(shard), ends_in_run=bool(n and shard[idx[n - 1]] == RS and ok), all_ws=bool(n == 0 and ok))


def fold_carries(carries, comma):
    """each rank's depth_in (comma) or run_in (RS)"""
    out, depth, run = [], 0, False
    for c in carries:
        out.append(depth if comma else run)
        if comma:
            depth += c["net"]
        else:
            run = c["ends_in_run"] or (run and c["all_ws"])
    return out


def filter_shard(shard, idx, n, comma, carry_in):
    """filter_pass_kernel over one shard: (filtered entries, separators, last separator)"""
    L = len(shard)
    vals, seps, last = [], 0, 0
    idx = [int(i) for i in idx[:n]]
    if comma:
        depth = carry_in
        for at in idx:
            c = shard[at]
            if c in (ord("{"), ord("[")):
                depth += 1
            elif c in (ord("}"), ord("]")):
                depth -= 1
            elif c == ord(",") and depth == 0:
                seps += 1
                last = max(last, at)
                continue
            vals.append(at)
        return vals, seps, last

    def glued(v, j0):
        if v < L and S.role(shard[v]) == 0:
            j = j0
            while j < n and idx[j] < v:
                j += 1
            if not (j < n and idx[j] == v):
                vals.append(v)

    if carry_in:  # the lead step
        v = 0
        while v < L and _ws_rs(shard[v]):
            if shard[v] == RS:
                seps += 1
                last = max(last, v)
            v += 1
        glued(v, 0)
    for i, at in enumerate(idx):
        if shard[at] != RS:
            vals.append(at)
            continue
        if i == 0 and carry_in and all(_ws_rs(c) for c in shard[:at]):
            continue
        if i > 0 and shard[idx[i - 1]] == RS and all(_ws_rs(c) for c in shard[idx[i - 1] + 1: at]):
            continue
        s, lst, v = 1, at, at + 1
        while v < L and _ws_rs(shard[v]):
            if shard[v] == RS:
                s += 1
                lst = v
            v += 1
        seps += s
        last = max(last, lst)
        glued(v, i + 1)
    return vals, seps, last


def walk(shard, arr):
    """stream_summary_kernel's words over the entries arr (as sjb200_stream_summary fields)"""
    k = len(arr)
    roles = [S.role(shard[i]) for i in arr]
    start, nobj, narr = -1, 0, 0
    for i in range(k - 1, 0, -1):
        if S.starts(roles[i], roles[i - 1]):
            start = i
            break
    for x in roles[max(start, 0):]:
        nobj += (x == 2) - (x == 3)
        narr += (x == 4) - (x == 5)
    return dict(count=k, len=len(shard), first_byte=int(arr[0]) if k else 0, last_byte=int(arr[-1]) if k else 0, start_index=max(start, 0),
                start_byte=int(arr[start]) if start >= 0 else 0, net_obj=nobj, net_arr=narr, role_first=roles[0] if k else 0,
                role_last=roles[-1] if k else 0, has_start=int(start >= 0))


def model(oracle, buf, cuts, mode):
    """every rank's view of a pass: (summaries for sjb200_delimited_fold, final_state, flags_all, per-rank scanned
    indexes, per-rank filtered entries, shards), or None when the last shard's trim differs from the whole buffer's"""
    sh = oracle.shards(buf, cuts, mode)
    if sh is None:
        return None
    state, scans = 0, []
    for s in sh:
        k, idx, state = oracle.scan(s, state)
        scans.append(idx)
    whole = b"".join(sh)
    unclosed = bool(state & 2)
    flags = 0 if oracle.port.validate_utf8(whole) else 1
    if oracle.port.stage1(whole, O.STREAMING_FINAL).err == O.UNESCAPED_CHARS:
        flags |= 2
    holder = max([r for r, idx in enumerate(scans) if len(idx)] or [-1])
    comma = not is_rs_mode(mode)
    ns = [len(idx) - (1 if unclosed and r == holder else 0) for r, idx in enumerate(scans)]
    carries = [carry(s, idx, n, comma) for s, idx, n in zip(sh, scans, ns)]
    cin = fold_carries(carries, comma)
    sums, filt = [], []
    for s, idx, n, c in zip(sh, scans, ns, cin):
        vals, seps, last = filter_shard(s, idx, n, comma, c)
        below = sum(1 for v in vals if v < last) if seps else 0
        sums.append(dict(count=len(idx), len=len(s), filtered=len(vals), seps=seps, last_sep=last, below=below, walk=walk(s, vals),
                         walk_below=walk(s, vals[:below]) if mode == O.COMMA_DELIMITED_PARTIAL else {}))
        filt.append(np.array(vals, dtype=np.uint32))
    return sums, state, flags, scans, filt, sh


def check(buf, cuts, mode, want, ranks):
    """ranks[r] = dict(err, n, kept, bytes_before, total_bytes, first_starts_document, filtered, filtered_before, words,
    tail): words = the rank's d_idx[0:filtered] after the pass.  want = port.stage1(whole buffer, mode)."""
    tag = (len(buf), cuts, mode)
    for r, g in enumerate(ranks):
        assert g["err"] == want.err, (tag, r, g["err"], want.err)
        assert g["bytes_before"] == cuts[r], (tag, r)
    if not want.wrote:
        for r, g in enumerate(ranks):
            assert g["n"] == 0 and g["kept"] == 0, (tag, r)
        return
    n = want.n
    fb = 0
    parts = []
    for r, g in enumerate(ranks):
        assert g["n"] == n, (tag, r, g["n"], n)
        assert g["filtered_before"] == fb, (tag, r)
        assert g["kept"] == min(max(n - fb, 0), g["filtered"]), (tag, r, g["kept"])
        w = np.asarray(g["words"], dtype=np.uint32)[: g["kept"]]
        parts.append(w + np.uint32(g["bytes_before"] & 0xFFFFFFFF))
        fb += g["filtered"]
    parts.append(np.asarray(ranks[0]["tail"], dtype=np.uint32))
    assert all(list(g["tail"]) == list(ranks[0]["tail"]) for g in ranks), tag
    G = np.concatenate(parts)
    assert np.array_equal(G[: n + 3], want.idx[: n + 3]), (tag, G[: n + 3][-6:], want.idx[: n + 3][-6:])
    if mode in (O.JSON_SEQUENCE_FINAL, O.COMMA_DELIMITED_FINAL):
        assert all(g["total_bytes"] == int(want.idx[n]) for g in ranks), tag
    starts_all = set(S.doc_starts(np.frombuffer(bytes(buf), dtype=np.uint8), want.idx, n))
    fb = 0
    for r, g in enumerate(ranks):
        if g["kept"]:
            assert bool(g["first_starts_document"]) == (fb in starts_all), (tag, r)
        fb += g["filtered"]


def rng_for(mode, salt):
    return random.Random(corpus.SEED ^ (salt + mode))
