"""CPU check of the pure host folds of a sharded grammar pass (sjb200_grammar_edge_fold, sjb200_grammar_result_fold):
the halo of every rank against the gathered stream, across ranks with 0, 1 and 2 structurals; the verdicts every rank
must share; and the owner of a document that spans ranks taking the first error over them."""
import ctypes as C
import random

import simdjson_b200 as sj
from simdjson_b200 import capi

NONE64 = (1 << 64) - 1
FAILED, BAD, WHOLE, FIRST, LAST = 1, 2, 4, 8, 16


def _edges(types, starts, cuts, whole, md=1024, flags=None):
    """the edge words of every rank for a gathered stream of token types and document starts"""
    es = (capi.GrammarEdge * (len(cuts) - 1))()
    for r in range(len(cuts) - 1):
        lo, hi = cuts[r], cuts[r + 1]
        t = types[lo:hi]
        n = hi - lo
        loc = [s - lo for s in starts if lo <= s < hi] if not whole else []
        b = [t[0] if n else 0xFF, t[1] if n >= 2 else 0xFF, t[n - 2] if n >= 2 else 0xFF, t[n - 1] if n else 0xFF]
        f = (WHOLE if whole else 0) | (FIRST if loc and loc[0] == 0 else 0) | (LAST if loc and loc[-1] == n - 1 else 0)
        es[r] = capi.GrammarEdge(n, len(loc), f | (flags[r] if flags else 0), md, b[0] | b[1] << 8 | b[2] << 16 | b[3] << 24, loc[0] if loc else 0)
    return es


def _fold(es):
    res, ranks = capi.GrammarEdgeFoldResult(), (capi.GrammarRank * len(es))()
    rc = sj.lib().sjb200_grammar_edge_fold(len(es), es, C.byref(res), ranks)
    return rc, res, ranks


def test_halo_matches_the_gathered_stream():
    rng = random.Random(7)
    alphabet = b'{}[]:,"dtl'
    for _ in range(400):
        N = rng.randrange(0, 12)
        types = [rng.choice(alphabet) for _ in range(N)]
        whole = rng.random() < 0.5
        starts = sorted(set(rng.sample(range(N), rng.randrange(0, N + 1)))) if N and not whole else []
        world = rng.randrange(1, 9)
        cuts = sorted([0, N] + [rng.randrange(0, N + 1) for _ in range(world - 1)])
        rc, res, ranks = _fold(_edges(types, starts, cuts, whole))
        assert rc == 0 and res.n == N and res.ndocs == (1 if whole else len(starts))
        is_start = (lambda k: k == 0) if whole else (lambda k: k == 0 or k in starts)
        for r in range(world):
            lo, hi, k = cuts[r], cuts[r + 1], ranks[r]
            assert k.tokens_before == lo and k.holds_root == (lo == 0 and hi > 0)
            assert k.owned == ((1 if r == 0 else 0) if whole else len([s for s in starts if lo <= s < hi]))
            if hi == lo:
                continue
            t = lambda j: types[j] if 0 <= j < N else 0xFF  # noqa: E731
            assert k.halo_before == (t(lo - 2) | t(lo - 1) << 8 | 0xFFFF0000), (types, cuts, r)
            assert k.halo_after == t(hi)
            want = (1 if lo >= 1 and is_start(lo - 1) else 0) | (2 if hi < N and is_start(hi) else 0) | (4 if lo == 0 else 0)
            assert k.halo_flags == want, (types, starts, cuts, r, k.halo_flags, want)
            assert k.last_type == t(N - 1)


def test_verdicts_every_rank_shares():
    types, cuts = list(b"[1,2]"), [0, 2, 5]
    assert _fold(_edges(types, [], cuts, True))[0] == 0
    assert _fold(_edges(types, [], cuts, True, flags=[0, FAILED]))[0] == sj.UNEXPECTED_ERROR
    es = _edges(types, [], cuts, True)
    es[1].max_depth = 0
    assert _fold(es)[0] == sj.CAPACITY
    es = _edges(types, [], cuts, True)
    es[1].max_depth = 512
    assert _fold(es)[0] == sj.UNEXPECTED_ERROR
    es = _edges(types, [], cuts, True)
    es[1].flags &= ~WHOLE
    assert _fold(es)[0] == sj.UNEXPECTED_ERROR
    rc, res, _ = _fold(_edges(types, [0], cuts, False, flags=[0, BAD]))
    assert rc == 0 and res.bad_table == 1


def test_spanning_document_takes_the_first_error():
    # documents at 0 (rank 0), 4 (rank 2); rank 1 is inside the first document, rank 3 inside the second
    types, starts, cuts = [ord("[")] * 8, [0, 4], [0, 2, 4, 6, 8]
    es = _edges(types, starts, cuts, False)
    t = (capi.GrammarTally * 4)()
    key = lambda i, c: i << 8 | c  # noqa: E731
    for r in range(4):
        t[r] = capi.GrammarTally(NONE64, NONE64, NONE64, 0, 0xFFFFFFFF)
    t[1].lead = key(3, 3)
    t[3].lead = key(7, 4)
    t[2].last = key(9, 3)  # its own structurals judge the end later than rank 3's leading error
    out, last = capi.ShardedDocumentErrorsResult(), (capi.ShardedDocumentError * 4)()
    assert sj.lib().sjb200_grammar_result_fold(4, es, t, C.byref(out), last) == 0
    assert (last[0].error, last[0].index) == (3, 3) and (last[2].error, last[2].index) == (4, 7)
    assert out.ndocs == 2 and out.ndocs_in_error == 2 and out.first_doc_in_error == 0 and out.first_error_index == 3
    t[1].lead = NONE64
    t[3].lead = NONE64
    t[2].last = NONE64
    assert sj.lib().sjb200_grammar_result_fold(4, es, t, C.byref(out), last) == 0
    assert (last[0].error, last[0].index) == (0, 4) and (last[2].error, last[2].index) == (0, 8)
    assert out.ndocs_in_error == 0 and out.first_doc_in_error == NONE64


def test_whole_empty_stream_is_empty():
    es = _edges([], [], [0, 0, 0], True)
    t = (capi.GrammarTally * 2)(*[capi.GrammarTally(NONE64, NONE64, NONE64, 0, 0xFFFFFFFF)] * 2)
    out, last = capi.ShardedDocumentErrorsResult(), (capi.ShardedDocumentError * 2)()
    assert sj.lib().sjb200_grammar_result_fold(2, es, t, C.byref(out), last) == 0
    assert (last[0].error, last[0].index) == (sj.EMPTY, 0) and out.first_doc_in_error == 0 and out.first_error == sj.EMPTY
