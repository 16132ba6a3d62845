"""The host fold of sharded stream passes (sjb200_stream_fold), driven without a GPU: every shard's summary is built from
the oracle's scan of the shard with its true incoming state, the fold's error, n, kept counts and rewrites are applied to
the oracle's shard indexes, and the gathered array must reproduce stage1(whole buffer, mode) in modes 0, 1 and 2."""
import random

import numpy as np
import pytest

import oracle_lib as O
import stream_shards as S
from simdjson_b200 import corpus, sharding


@pytest.fixture(scope="module")
def oracle():
    return S.Oracle()


def fold_ranks(oracle, buf, cuts, mode):
    """per-rank results of a pass as the fold gives them, the rank's words rewritten as finish() rewrites them"""
    got = oracle.summaries(buf, cuts, mode)
    if got is None:
        return None
    sums, final_state, flags, idxs = got
    err, n_written, n, total, ranks = sharding.fold_stream(mode, final_state, flags, sums)
    out = []
    for r, (s, x) in enumerate(zip(sums, ranks)):
        words = np.concatenate([idxs[r], np.array([s["len"], s["len"], 0] if r == len(sums) - 1 else [], dtype=np.uint32)]).astype(np.uint32)
        if not n_written:
            assert not x["rewrites"] and x["kept"] == 0
        for pos, val in x["rewrites"]:
            words[pos] = val
        out.append(dict(err=err, n=n if n_written else 0, kept=x["kept"], bytes_before=x["bytes_before"], total_bytes=total,
                        first_starts_document=x["first_starts_document"], count=s["count"], words=words))
    return out


@pytest.mark.parametrize("mode", [O.REGULAR, O.STREAMING_PARTIAL, O.STREAMING_FINAL])
def test_fold_reproduces_whole_stage1(oracle, mode):
    rng = random.Random(corpus.SEED ^ (0x5F0 + mode))
    checked, skipped, rewrites_across = 0, 0, 0
    errors = set()
    for name, buf in S.inputs(rng):
        want = oracle.port.stage1(buf, mode)
        for world in (1, 2, 4, 8):
            for cuts in S.cut_sets(rng, buf, world, 6 if len(buf) > 100 else 3):
                ranks = fold_ranks(oracle, buf, cuts, mode)
                if ranks is None:
                    skipped += 1
                    continue
                S.check(buf, cuts, mode, want, ranks)
                checked += 1
                errors.add(want.err)
    assert checked > 1000 and skipped < checked // 20, (checked, skipped)
    if mode != O.REGULAR:
        assert {O.SUCCESS, O.EMPTY} <= errors, errors


def test_fold_special_cases(oracle):
    """a stream whose last string opens several shards before the end; a last shard that is one partial character; a cut
    right after an opening bracket; shards without structurals"""
    buf = b'{"a":1} [2] "' + b"x y " * 50
    cuts = [0, 5, 13, 60, 100, 140, 170, 190, len(buf)]
    for mode in (O.REGULAR, O.STREAMING_PARTIAL, O.STREAMING_FINAL):
        S.check(buf, cuts, mode, oracle.port.stage1(buf, mode), fold_ranks(oracle, buf, cuts, mode))
    buf = b'{"a":[1,2]} [3]\xf0\x9f\x98'
    for mode in (O.STREAMING_PARTIAL, O.STREAMING_FINAL):
        cuts = [0, 6, len(buf) - 3, len(buf)]
        ranks = fold_ranks(oracle, buf, cuts, mode)
        assert ranks[-1]["count"] == 0 and ranks[-1]["words"][:3].tolist() == ([0, 0, 0] if mode == O.STREAMING_PARTIAL else ranks[-1]["words"][:3].tolist())
        S.check(buf, cuts, mode, oracle.port.stage1(buf, mode), ranks)
    # one rank only, the partial character: trims to nothing
    buf = b"\xe2\x82"
    for mode in (O.STREAMING_PARTIAL, O.STREAMING_FINAL):
        ranks = fold_ranks(oracle, buf, [0, 2], mode)
        assert ranks[0]["err"] == O.UTF8_ERROR and ranks[0]["n"] == 0
