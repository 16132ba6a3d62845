"""CPU check of the pure host fold of a sharded pointer pass (sjb200_pointer_edge_fold): every rank's bases, holders,
halo type and the document that holds its last structural -- whether it goes on past the rank, its structurals on later
ranks and the first token in error of those pieces -- against the gathered stream, across ranks with 0, 1 and 2
structurals; and the verdicts every rank must share."""
import ctypes as C
import random

import simdjson_b200 as sj
from simdjson_b200 import capi

NONE64 = (1 << 64) - 1
FAILED, BAD, WHOLE, OVER = 1, 2, 4, 8


def _edges(types, starts, cuts, whole, np_=4, hashes=None, flags=None, errors=None):
    """the edge words of every rank for a gathered stream of token types (0: a token in error, its code in errors) and
    document starts"""
    errors = errors or {}
    es = (capi.PointerEdge * (len(cuts) - 1))()
    for r in range(len(cuts) - 1):
        lo, hi = cuts[r], cuts[r + 1]
        n = hi - lo
        loc = [s - lo for s in starts if lo <= s < hi] if not whole else []
        lead_end = loc[0] if loc else n
        lead = next((k for k in range(lead_end) if types[lo + k] == 0), 0xFFFFFFFF)
        t = (types[lo] | types[hi - 1] << 8) if n else 0xFFFF
        es[r] = capi.PointerEdge(n, len(loc), (WHOLE if whole else 0) | (flags[r] if flags else 0), np_, hashes[r] if hashes else 77, t, lead_end, lead,
                                 errors.get(lo + lead, 0) if lead != 0xFFFFFFFF else 0)
    return es


def _fold(es):
    res, ranks = capi.PointerEdgeFoldResult(), (capi.PointerRank * len(es))()
    rc = sj.lib().sjb200_pointer_edge_fold(len(es), es, C.byref(res), ranks)
    return rc, res, ranks


def _want(types, starts, cuts, whole, errors):
    """per rank, from the gathered stream: (tokens_before, docs_before, owned, walks, prev, next, next_type, lead_owner,
    tail_owner, continues, after, tail_error, tail_error_index)"""
    N, R = len(types), len(cuts) - 1
    rank_of = lambda k: max(r for r in range(R) if cuts[r] <= k < cuts[r + 1])  # noqa: E731
    docs = [(0, N)] if whole and N else ([] if whole else [(s, starts[i + 1] if i + 1 < len(starts) else N) for i, s in enumerate(starts)])
    doc_of = lambda k: next((i for i, (s, e) in enumerate(docs) if s <= k < e), None)  # noqa: E731
    owner = lambda d: 0 if whole else rank_of(docs[d][0])  # noqa: E731
    out = []
    for r in range(R):
        lo, hi = cuts[r], cuts[r + 1]
        n = hi - lo
        holders = [q for q in range(R) if cuts[q + 1] > cuts[q]]
        prev = max([q for q in holders if q < r], default=-1)
        nxt = min([q for q in holders if q > r], default=-1)
        owned = (1 if r == 0 else 0) if whole else sum(1 for s in starts if lo <= s < hi)
        walks = (1 if n and lo == 0 else 0) if whole else (owned if n else 0)
        lead_owner = tail_owner = -1
        cont, after, terr, tidx = 0, 0, 0, NONE64
        if n:
            d0 = doc_of(lo)
            if d0 is not None and docs[d0][0] < lo:
                lead_owner = owner(d0)
            dl = doc_of(hi - 1)
            if dl is not None:
                tail_owner = owner(dl)
                s, e = docs[dl]
                if e > hi:
                    cont, after = 1, e - hi
                    k = next((k for k in range(hi, e) if types[k] == 0), None)
                    if k is not None:
                        terr, tidx = errors.get(k, 0), k
        out.append((lo, sum(1 for s in starts if s < lo) if not whole else min(r, 1), owned, walks, prev, nxt, types[cuts[nxt]] if nxt >= 0 else 0xFF,
                    lead_owner, tail_owner, cont, after, terr, tidx))
    return out


def test_ranks_match_the_gathered_stream():
    rng = random.Random(11)
    alphabet = [ord(c) for c in '{}[]:,"dtl'] + [0]
    for _ in range(600):
        N = rng.randrange(0, 14)
        types = [rng.choice(alphabet) for _ in range(N)]
        errors = {k: rng.choice([10, 13, 30]) for k in range(N) if types[k] == 0}
        whole = rng.random() < 0.4
        starts = [] if whole else sorted(rng.sample(range(N), rng.randrange(0, N + 1))) if N else []
        R = rng.randrange(1, 9)
        cuts = [0] + sorted(rng.randrange(0, N + 1) for _ in range(R - 1)) + [N]
        rc, res, ranks = _fold(_edges(types, starts, cuts, whole, errors=errors))
        assert rc == 0 and res.error == 0 and res.n == N and res.bad_table == 0
        assert res.ndocs == (1 if whole else len(starts))
        for r, w in enumerate(_want(types, starts, cuts, whole, errors)):
            k = ranks[r]
            got = (k.tokens_before, k.docs_before, k.owned, k.walks, k.prev_holder, k.next_holder, k.next_type, k.lead_owner, k.tail_owner,
                   k.tail_continues, k.tail_after, k.tail_error, k.tail_error_index)
            assert got == w, (types, starts, cuts, whole, r, got, w)


def test_verdicts_every_rank_shares():
    types = [ord("[")] * 3 + [ord("]")] * 3
    cuts = [0, 2, 4, 6]
    ok = _edges(types, [0, 3], cuts, False)
    assert _fold(ok)[0] == 0
    for flags, hashes, np_, want in (([0, FAILED, 0], None, 4, sj.UNEXPECTED_ERROR), ([0, 0, OVER], None, 4, sj.CAPACITY),
                                     ([FAILED, OVER, 0], None, 4, sj.UNEXPECTED_ERROR), (None, [77, 78, 77], 4, sj.UNEXPECTED_ERROR),
                                     (None, None, 1025, sj.CAPACITY), ([0, WHOLE, 0], None, 4, sj.UNEXPECTED_ERROR)):
        rc, res, _ = _fold(_edges(types, [0, 3], cuts, False, np_, hashes, flags))
        assert rc == res.error == want, (flags, hashes, np_)
    rc, res, _ = _fold(_edges(types, [0, 3], cuts, False, flags=[0, BAD, 0]))
    assert rc == 0 and res.bad_table == 1  # a bad table fails the pass after its results are written
    rc, res, _ = _fold(_edges(types, [], cuts, True, flags=[0, BAD, 0]))
    assert rc == 0 and res.bad_table == 0  # whole mode has no table
