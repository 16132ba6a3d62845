"""The host fold of sharded RS-delimited and comma-delimited passes (sjb200_delimited_fold), driven without a GPU: every
shard is scanned by the oracle with its true incoming state, a Python model of the carry and filter rounds
(delimited_shards.py) gives every rank's filter totals and walks, the fold's error, n, kept counts and tail words are
applied, and the gathered array must reproduce stage1(whole buffer, mode) word for word in modes 3-6."""
import numpy as np
import pytest

import delimited_shards as D
import oracle_lib as O
from simdjson_b200 import sharding


@pytest.fixture(scope="module")
def oracle():
    import stream_shards as S
    return S.Oracle()


def fold_ranks(oracle, buf, cuts, mode):
    """per-rank results of a pass as the fold gives them, or None (see delimited_shards.model)"""
    got = D.model(oracle, buf, cuts, mode)
    if got is None:
        return None
    sums, final_state, flags, scans, filt, sh = got
    err, n_written, n, total, tail, ranks = sharding.fold_delimited(mode, final_state, flags, sums)
    words = []
    for t in tail:
        if t[0] == "value":
            words.append(t[1])
        else:
            kind, r, pos = t
            src = filt[r] if kind == "filtered" else scans[r]
            words.append((int(src[pos]) + ranks[r]["bytes_before"]) & 0xFFFFFFFF)
    out = []
    for r, x in enumerate(ranks):
        if not n_written:
            assert x["kept"] == 0
        out.append(dict(err=err, n=n if n_written else 0, kept=x["kept"], bytes_before=x["bytes_before"], total_bytes=total,
                        first_starts_document=x["first_starts_document"], filtered=len(filt[r]), filtered_before=x["filtered_before"],
                        words=filt[r], tail=words))
    return out


@pytest.mark.parametrize("mode", D.MODES)
def test_fold_reproduces_whole_stage1(oracle, mode):
    rng = D.rng_for(mode, 0xDE1)
    checked, skipped = 0, 0
    errors = set()
    for name, buf, modes in D.inputs(rng):
        if mode not in modes:
            continue
        want = oracle.port.stage1(buf, mode)
        for world in (1, 2, 4, 8):
            for cuts in D.cut_sets(rng, buf, world, 14 if len(buf) > 100 else 5):
                ranks = fold_ranks(oracle, buf, cuts, mode)
                if ranks is None:
                    skipped += 1
                    continue
                D.check(buf, cuts, mode, want, ranks)
                checked += 1
                errors.add(want.err)
    assert checked > 1000 and skipped < checked // 20, (checked, skipped)
    want_errors = {O.SUCCESS, O.EMPTY} | ({O.CAPACITY} if mode in (O.JSON_SEQUENCE_PARTIAL, O.COMMA_DELIMITED_PARTIAL) else set())
    assert want_errors <= errors, errors


def test_fold_special_cases(oracle):
    """cuts placed by hand: a run of RS / whitespace spanning whole shards, a scalar glued to a run's last RS at a shard's
    byte 0, root commas in shards entered at a non-zero or negative depth, a string whose quote is dropped on a rank before the last, a
    last shard that is one partial character, old word m an unfiltered leftover on another rank"""
    cases = [
        (b"\x1e[1]\n\x1e  \x1e   \x1e  \x1e42\x1e\n", [0, 6, 9, 12, 16, 19]),           # run over 4 cuts, "42" glued at byte 0 of a shard
        (b"\x1e[1]\n\x1e" + b" " * 40 + b"\x1e7", [0, 10, 30, 46, 47]),               # whole shards of whitespace, glued 7 alone
        (b"\x1e1\x1e \x1e2", [0, 2, 3, 6]),                                           # 1\x1e: an RS glued behind a scalar starts no run
        (b"[1,[2]],{}]],{},3", [0, 8, 12, 17]),                                        # shards entered at depths 0, 0, -2
        (b"{\"a\":1},[2],\"x, y, z", [0, 9, 14, 18, 21]),                              # the dropped quote on rank 1 of 4
        (b"\x1e{\"a\":1}\n\x1e\"x y z", [0, 10, 13, 17]),
        (b"\x1e[1]\n\x1e[2]\xf0\x9f\x98", [0, 5, 9]),                                  # the last shard only a partial character
        (b"[1,2],{\"a\":3}\xe2\x82", [0, 6, 13, 15]),
        (b"\x1e[1,2,3]\n\x1e{\"b\":[4,5]}\n", [0, 3, 12, 20, 26]),                    # final: old word m = a scanned RS on rank 1
    ]
    for buf, cuts in cases:
        cuts = [c for c in cuts if c < len(buf)] + [len(buf)]  # (the last cut is the end)
        modes = D.MODES[:2] if buf[:1] == b"\x1e" else D.MODES[2:]
        for mode in modes:
            ranks = fold_ranks(oracle, buf, cuts, mode)
            assert ranks is not None, (buf, cuts)
            D.check(buf, cuts, mode, oracle.port.stage1(buf, mode), ranks)
    # one rank only, the partial character: trims to nothing
    for mode in D.MODES:
        ranks = fold_ranks(oracle, b"\xe2\x82", [0, 2], mode)
        assert ranks[0]["err"] == O.UTF8_ERROR and ranks[0]["n"] == 0


def test_old_word_m_is_a_leftover_on_another_rank(oracle):
    """final modes: word n+1 (the old word n) is a scanned structural the in-place filter left behind, held by a rank
    other than the last -- RS runs with several RS entries leave the filtered array shorter than the scan"""
    rng = D.rng_for(0, 0x01D)
    seen = 0
    for k in range(60):
        docs = [b"[%d]" % k, b'{"a":%d}' % k, b"%d" % k, b'"s"']
        buf = b"".join(b"\x1e" + b" \x1e" * rng.randrange(0, 3) + b"\n" * rng.randrange(0, 2) + rng.choice(docs) for _ in range(8))
        want = oracle.port.stage1(buf, O.JSON_SEQUENCE_FINAL)
        for cuts in D.cut_sets(rng, buf, 4, 6):
            got = D.model(oracle, buf, cuts, O.JSON_SEQUENCE_FINAL)
            if got is None:
                continue
            tail = sharding.fold_delimited(O.JSON_SEQUENCE_FINAL, got[1], got[2], got[0])[4]
            seen += tail[1][0] == "scanned" and tail[1][1] < 3
            D.check(buf, cuts, O.JSON_SEQUENCE_FINAL, want, fold_ranks(oracle, buf, cuts, O.JSON_SEQUENCE_FINAL))
    assert seen > 0
