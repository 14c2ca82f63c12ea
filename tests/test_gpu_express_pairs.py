"""GPU parity of the express tokenizer kernel (csrc/sp_encode.cu: sp_express_kernel), bit-exact against the CPU
oracle, at the seams between the requests of a batch: batches smaller than the grid, neighbouring requests of very
different lengths (empty, one word, 16 KB), a hand-over, a long word or a hard word in one request while its
neighbours stay in the kernel, and a truncating ids_stride in some requests only.  Every case runs at the default
grid and at one block per SM, where every warp takes many requests in turn from the task counter."""
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
MODEL_8K = os.path.join(HERE, "golden", "sp_bpe_8k")
MODEL_32K = os.path.join(HERE, "golden", "sp_natural_32k")


@pytest.fixture(scope="module", params=[MODEL_8K, MODEL_32K], ids=["bpe8k", "natural32k"])
def pair(request, oracle):
    import xllm_service_b200 as x
    h = x.Ingest(tokenizer_path=request.param)
    yield h, oracle.SentencePieceOracle(request.param)
    h.close()


@pytest.fixture(params=["default", "one_block_per_sm"])
def grid(request, monkeypatch):
    if request.param == "one_block_per_sm":
        monkeypatch.setenv("XLLM_SP_EXPRESS_BLOCKS_PER_SM", "1")
    yield request.param


def _words(rnd, n, lo=1, hi=9, alphabet="abcdefghijklmnopqrstuvwxyz"):
    return ["".join(rnd.choice(alphabet) for _ in range(rnd.randint(lo, hi))) for _ in range(n)]


def _text(rnd, nbytes):
    out, size = [], 0
    while size < nbytes:
        w = _words(rnd, 1, 1, 9)[0]
        out.append(w)
        size += len(w) + 1
    return " ".join(out).encode()[:nbytes]


def _check(tok, orc, texts, stride=None):
    """Full rows must match the oracle; a row the stride truncates holds the oracle's prefix, with the full count."""
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    if stride is None:
        stride = max(16, 2 * max((len(t) for t in texts), default=0) + 16)
    ids, n_ids, status = tok.encode_batch(b.text, b.offsets, stride)
    bad = []
    for i, t in enumerate(texts):
        want = orc.encode(t).tolist()
        keep = min(len(want), stride)
        if (int(n_ids[i]) != len(want) or int(status[i]) != (1 if len(want) > stride else 0)
                or ids[i, :keep].tolist() != want[:keep]):
            bad.append((i, len(t), int(n_ids[i]), len(want), int(status[i]), t[:32]))
    assert not bad, bad[:5]
    return status


@pytest.mark.parametrize("n", [1, 2, 3, 5, 33])
def test_small_batches(pair, grid, n):
    tok, orc = pair
    rnd = random.Random(100 + n)
    texts = [_text(rnd, rnd.choice([7, 300, 1500, 5000])) for _ in range(n)]
    _check(tok, orc, texts)


def test_neighbours_of_very_different_lengths(pair, grid):
    tok, orc = pair
    rnd = random.Random(5)
    big = _text(rnd, 16384)
    texts = []
    for _ in range(6):
        texts += [b"", b"word", big, b" ", _text(rnd, 16384), b"a", b"", _text(rnd, 700)]
    _check(tok, orc, texts)


def test_hand_over_in_one_request(pair, grid):
    tok, orc = pair
    rnd = random.Random(9)
    texts = []
    for k in range(12):
        for sp in ("é", "日本", "\xa0"):
            head = " ".join(_words(rnd, rnd.randint(1, 400)))
            texts.append(_text(rnd, rnd.randint(100, 6000)))
            texts.append((head + " " + sp + " " + " ".join(_words(rnd, rnd.randint(1, 200)))).encode())
    _check(tok, orc, texts)


def test_long_or_hard_word_in_one_request(pair, grid):
    tok, orc = pair
    rnd = random.Random(13)
    odd = ["".join(rnd.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(n)) for n in (16, 40, 300)]
    odd += ["{}[]{}[]{}[]{}", "Q9z~X8y`W7v^U6t"]
    texts = []
    for o in odd:
        for k in (0, 5, 40, 200):
            texts.append(_text(rnd, rnd.randint(200, 4000)))
            texts.append((" ".join(_words(rnd, k)) + " " + o + " " + " ".join(_words(rnd, 300))).strip().encode())
    _check(tok, orc, texts)


def test_truncating_stride_in_one_request(pair, grid):
    tok, orc = pair
    rnd = random.Random(17)
    stride = 96
    texts = []
    for i in range(40):
        # short requests fit the row; every fourth one is far longer than the row and is truncated
        texts.append(_text(rnd, 3000 + 37 * i) if i % 4 == 1 else _text(rnd, rnd.randint(0, 80)))
    status = _check(tok, orc, texts, stride=stride)
    assert (status == 1).sum() >= 10 and (status == 0).sum() >= 10
