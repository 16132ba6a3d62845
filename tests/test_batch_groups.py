"""sjb200_stage1_dev_batch with several documents per scan launch: every document's result must equal a call of its
own, in every mode, whatever mix of sizes, alignments and early errors shares the launch."""
import random

import numpy as np
import pytest
import torch

import oracle_lib as O
import simdjson_b200 as sj
from test_gpu_parity import TILE, _big_adversarial

pytestmark = pytest.mark.gpu
CAP = 2 << 20


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


def _dev(b, offset=0):
    """b on the device at `offset` bytes past a 256-byte aligned allocation (offset % 16 != 0: no TMA)"""
    base = torch.zeros(len(b) + offset + 1, dtype=torch.uint8, device="cuda")
    view = base[offset: offset + len(b)]
    if len(b):
        view.copy_(torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()))
    return view


def _check(parser, port, docs, d_bufs, d_idxs, mode):
    res = parser.stage1_device_batch(d_bufs, d_idxs, mode)
    for i, (b, (err, n)) in enumerate(zip(docs, res)):
        if len(b) > CAP:  # beyond the parser's capacity (json_structural_indexer.h L195)
            assert err == sj.CAPACITY, (i, mode, err)
            continue
        want = port.stage1(b, mode)
        assert err == want.err, (i, len(b), mode, err, want.err)
        if want.wrote:
            assert n == want.n, (i, len(b), mode)
            got = d_idxs[i].cpu().numpy().view(np.uint32)[: n + 3]
            assert np.array_equal(got, want.words()), (i, len(b), mode)
    return res


def _mixed_docs(rng):
    """short, block-sized, element-sized and multi-element documents, some ending inside an element or a string"""
    docs = []
    for n in (17, 100, 4095, 4096, 4097, 2 * TILE, 2 * TILE + 1, 5 * TILE + 333, 40, 9 * TILE + 4000, 3000):
        docs.append(_big_adversarial(rng, n))
    docs.append(b'{"a": "unterminated \\" string' + b"x" * 70000)
    docs.append(b'[1, {"k": "\xc3\xa9\xe2\x82\xac"}, "\xf0\x9f\x98\x80"]' * 3000)
    docs.append(b'{"tail": "\xe2\x82')  # partial UTF-8 at the end
    return docs


@pytest.mark.parametrize("mode", range(7))
def test_many_documents_one_group(parser, port, mode):
    rng = random.Random(1000 + mode)
    docs = _mixed_docs(rng)
    docs = docs[:3] + [b"", b"x" * (CAP + 1)] + docs[3:]  # empty and over-capacity documents in the middle of a group
    offsets = [0 if i % 3 else 5 for i in range(len(docs))]  # TMA and plain-load buffers mixed
    d_bufs = [_dev(b, o) for b, o in zip(docs, offsets)]
    d_idxs = [torch.zeros(sj.lib().sjb200_index_words(max(len(b), 1)), dtype=torch.int32, device="cuda") for b in docs]
    launches = parser.get_stat("launches")
    _check(parser, port, docs, d_bufs, d_idxs, mode)
    if mode == sj.REGULAR:  # (the other modes add epilogue launches per document)
        assert parser.get_stat("launches") - launches < len(docs) - 2, "the documents should share scan launches"


def test_more_documents_than_one_launch_takes(parser, port):
    rng = random.Random(7)
    docs = [_big_adversarial(rng, rng.choice((1, 5, 300, 4096, TILE + 7))) for _ in range(150)]
    d_bufs = [_dev(b) for b in docs]
    d_idxs = [torch.zeros(sj.lib().sjb200_index_words(len(b)), dtype=torch.int32, device="cuda") for b in docs]
    _check(parser, port, docs, d_bufs, d_idxs, sj.REGULAR)
    parser.get_stat("kernel_ms_mean")
    _check(parser, port, docs, d_bufs, d_idxs, sj.STREAMING_FINAL)
    assert parser.get_stat("kernel_ms_mean") > 0


def test_shared_index_buffer_keeps_serial_order(parser, port):
    """the same index buffer for several documents with different inputs: it must hold what the last of them wrote"""
    docs = [b"[" + b'{"a": [1, 2, "x\\"y"]}, ' * k + b"0]" for k in (5000, 9, 3000, 4)]
    shared = torch.zeros(sj.lib().sjb200_index_words(max(len(b) for b in docs)), dtype=torch.int32, device="cuda")
    other = torch.zeros_like(shared)
    d_bufs = [_dev(b) for b in docs]
    for mode in (sj.REGULAR, sj.STREAMING_FINAL):
        d_idxs = [shared, other, shared, shared]
        res = parser.stage1_device_batch(d_bufs, d_idxs, mode)
        for b, (err, n) in zip(docs, res):
            want = port.stage1(b, mode)
            assert want.wrote and (err, n) == (want.err, want.n)
        want = port.stage1(docs[3], mode)
        assert np.array_equal(shared.cpu().numpy().view(np.uint32)[: want.n + 3], want.words())
        want = port.stage1(docs[1], mode)
        assert np.array_equal(other.cpu().numpy().view(np.uint32)[: want.n + 3], want.words())


def test_input_overwritten_by_an_earlier_output(parser, port):
    """a document whose input is another document's index output, in the same call: the scan sees the written indexes"""
    first = b'[1, 2, {"a": "b\\"c"}] ' * 4000
    d_first = _dev(first)
    words = sj.lib().sjb200_index_words(len(first))
    out = torch.zeros(words, dtype=torch.int32, device="cuda")
    second_len = 4096
    second_view = out.view(torch.uint8)[:second_len]
    res = parser.stage1_device_batch([d_first, second_view], [out, torch.zeros(words, dtype=torch.int32, device="cuda")], sj.STREAMING_FINAL)
    want_first = port.stage1(first, sj.STREAMING_FINAL)
    assert res[0][0] == want_first.err and want_first.wrote
    buf = np.zeros(words, dtype=np.uint32)
    buf[: want_first.n + 3] = want_first.words()
    want_second = port.stage1(buf.view(np.uint8)[:second_len].tobytes(), sj.STREAMING_FINAL)
    assert res[1][0] == want_second.err
