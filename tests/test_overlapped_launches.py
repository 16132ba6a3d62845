"""sjb200_stage1_dev_batch with consecutive scan launches that overlap (programmatic dependent launch, option pdl): a
launch starts while the previous one still runs, and waits for it before its first access that could conflict.  Every
case runs with pdl 0 and 1 and checks each document's error code, n and (n + 3) index words against the CPU oracle
and against one-by-one sjb200_stage1_dev calls -- including batches over 4 index arrays that every launch writes again,
documents so short that launches overlap most, and a launch whose input is what the previous launch wrote."""
import random

import numpy as np
import pytest
import torch

import oracle_lib as O
import simdjson_b200 as sj
from simdjson_b200 import corpus
from test_gpu_parity import _big_adversarial

pytestmark = pytest.mark.gpu
BIG = 64 << 20
CAP = BIG + 4096
MODES = (sj.REGULAR, sj.STREAMING_FINAL)


@pytest.fixture(scope="module")
def port():
    return O.Port()


@pytest.fixture(scope="module")
def parser():
    rc, p = sj.get_active_implementation().create_dom_parser_implementation(CAP)
    assert rc == sj.SUCCESS, sj.ERROR_NAMES.get(rc, rc)
    p.set_option("time_kernel", 1)
    yield p
    p.close()


def _words(t, n):
    return t.cpu().numpy().view(np.uint32)[: n + 3]


def _one_by_one(parser, d_bufs, mode):
    """each document through its own sjb200_stage1_dev call, in order, into a buffer of its own"""
    out = []
    for b in d_bufs:
        d_idx = torch.zeros(sj.lib().sjb200_index_words(max(b.numel(), 1)), dtype=torch.int32, device="cuda")
        parser.n_structural_indexes = 0  # (a call that stores no n leaves it as it was, the batch reports 0)
        rc = parser.stage1_device(b, mode, d_idx=d_idx)
        out.append((rc, parser.n_structural_indexes, d_idx))
    return out


def _check_batch(parser, port, d_bufs, d_idxs, mode, pdl, inputs=None):
    """the batch against the oracle; an index array shared by several documents must hold
    what the last of them wrote.  inputs[i]: the bytes document i reads (default: d_bufs[i] after the batch)"""
    parser.set_option("pdl", pdl)
    try:
        res = parser.stage1_device_batch(d_bufs, d_idxs, mode)
        torch.cuda.synchronize()
        if inputs is None:
            inputs = [bytes(b.cpu().numpy()) for b in d_bufs]
        last = {}  # index array -> the last document that writes it (what a document without a result leaves there is not checked)
        for i, (err, n) in enumerate(res):
            want = port.stage1(inputs[i], mode)
            assert err == want.err, (i, len(inputs[i]), mode, pdl, err, want.err)
            if want.wrote:
                assert n == want.n, (i, len(inputs[i]), mode, pdl, n, want.n)
            last[d_idxs[i].data_ptr()] = (i, want)
        for i, t in enumerate(d_idxs):
            j, want = last[t.data_ptr()]
            if j == i and want.wrote:
                assert np.array_equal(_words(t, want.n), want.words()), (i, len(inputs[i]), mode, pdl)
    finally:
        parser.set_option("pdl", 1)
    return res


def _against_one_by_one(parser, d_bufs, res, mode, d_idxs=None):
    """error code and n of every document, and the index words of d_idxs[i] where document i wrote them last"""
    for i, ((err, n), (rc1, n1, idx1)) in enumerate(zip(res, _one_by_one(parser, d_bufs, mode))):
        assert (err, n) == (rc1, n1), (i, mode, err, n, rc1, n1)
        if d_idxs is not None and n > 0 and all(t.data_ptr() != d_idxs[i].data_ptr() for t in d_idxs[i + 1:]):
            assert np.array_equal(_words(d_idxs[i], n), _words(idx1, n1)), (i, mode)


@pytest.fixture(scope="module")
def big_docs():
    return [corpus.random_json(BIG, seed=corpus.SEED + 7919 * k) for k in range(2)]


@pytest.mark.parametrize("pdl", (0, 1))
@pytest.mark.parametrize("mode", MODES)
def test_64mib_documents_into_four_shared_index_arrays(parser, port, big_docs, mode, pdl):
    d_docs = [torch.from_numpy(np.frombuffer(d, dtype=np.uint8).copy()).cuda() for d in big_docs]
    words = sj.lib().sjb200_index_words(BIG)
    d_idxs = [torch.zeros(words, dtype=torch.int32, device="cuda") for _ in range(4)]
    k = 10  # three launches of 4, 4 and 2 documents
    bufs = [d_docs[i % 2] for i in range(k)]
    idxs = [d_idxs[(i * 3) % 4] for i in range(k)]  # documents 0..3 write different arrays, 4..7 write them again
    inputs = [bytes(big_docs[i % 2]) for i in range(k)]
    res = _check_batch(parser, port, bufs, idxs, mode, pdl, inputs)
    _against_one_by_one(parser, bufs[:2], res[:2], mode)


def _valid_doc(n):
    """a valid document of about n bytes (its index words are checked whatever the mode)"""
    row = b'{"k": [1, 2.5, "s\\"q"], "u": "\xc3\xa9"}, '
    return b"0" if n < 2 else b"[]" if n < 30 else b"[" + row * ((n - 3) // len(row)) + b"0]"


def _small_docs(rng, count):
    """adversarial documents (mostly errors) and valid ones; the last document of each index array is valid"""
    sizes = (1, 2, 17, 100, 1000, 4095, 4097, 32768, 65537, 200000)
    docs = []
    for i in range(count):
        n = rng.choice(sizes)
        docs.append(_valid_doc(n) if i % 2 or i >= count - 4 else _big_adversarial(rng, n)[:n])
    return docs


@pytest.mark.parametrize("pdl", (0, 1))
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("count", (8, 61, 200))
def test_small_documents_into_four_shared_index_arrays(parser, port, mode, pdl, count):
    """short launches overlap most: 1 B to 200 KB per document, 4 per launch"""
    rng = random.Random(count * 31 + mode)
    docs = _small_docs(rng, count)
    d_bufs = [torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).cuda() for b in docs]
    words = sj.lib().sjb200_index_words(200000)
    d_idxs = [torch.zeros(words, dtype=torch.int32, device="cuda") for _ in range(4)]
    idxs = [d_idxs[i % 4] for i in range(count)]
    res = _check_batch(parser, port, d_bufs, idxs, mode, pdl, docs)
    _against_one_by_one(parser, d_bufs, res, mode, idxs)


@pytest.mark.parametrize("pdl", (0, 1))
@pytest.mark.parametrize("mode", MODES)
def test_input_written_by_the_previous_launch(parser, port, mode, pdl):
    """document C reads the end of the index array document A wrote in the launch before, E reads what C wrote: the
    launches of C and E must not read their input before the previous launch is done"""
    rng = random.Random(99 + mode)
    a = corpus.random_json(3 << 20, seed=corpus.SEED + 5)
    n_a = port.stage1(a, sj.REGULAR).n
    words = sj.lib().sjb200_index_words(len(a))
    fresh = lambda: torch.zeros(words, dtype=torch.int32, device="cuda")  # noqa: E731
    idx_a, idx_c, idx_e = fresh(), fresh(), fresh()
    others = [_big_adversarial(rng, n) for n in (5000, 70000, 300, 140000)]
    d_others = [torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).cuda() for b in others]
    tail = 64 << 10
    off = (4 * (n_a + 3) - tail) & ~15  # the words A's last elements and its sentinels write
    d_c = idx_a.view(torch.uint8)[off: off + tail]
    d_e = idx_c.view(torch.uint8)[: 8192]
    d_a = torch.from_numpy(np.frombuffer(a, dtype=np.uint8).copy()).cuda()
    bufs = [d_a, d_others[0], d_others[1], d_c, d_others[2], d_e, d_others[3]]
    idxs = [idx_a, fresh(), fresh(), idx_c, fresh(), idx_e, fresh()]
    res = _check_batch(parser, port, bufs, idxs, mode, pdl)
    _against_one_by_one(parser, bufs, res, mode, idxs)
