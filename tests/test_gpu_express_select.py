"""GPU parity of the express tokenizer kernel (csrc/sp_encode.cu: express_run), bit-exact against the CPU oracle,
where a step hands lane k its words k and k + 32: each lane's word starts packed from a table, the owner of word j
found from the lanes' first-start indices, and a word's end from the owner's and its successor's non-space bits.  So:
16-byte units holding 0 .. 8 word starts at every alignment, runs of units without a start, exactly 63 / 64 / 65
complete words with the 65th far from the 64th, words that end on the last byte of the next unit, words cut by the
window's last byte and texts that end there, steps that start inside a unit with starts on both sides of the
position, and a randomized sweep of start densities with the express kernel switched off as a second witness."""
import os
import random

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
MODELS = {"bpe8k": os.path.join(HERE, "golden", "sp_bpe_8k"), "natural32k": os.path.join(HERE, "golden", "sp_natural_32k")}


@pytest.fixture(scope="module", params=list(MODELS), ids=list(MODELS))
def model(request, oracle):
    import xllm_service_b200 as x
    h = x.Ingest(tokenizer_path=MODELS[request.param])
    yield request.param, h, oracle.SentencePieceOracle(MODELS[request.param])
    h.close()


def _check(tok, orc, texts):
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    stride = max(16, 14 * max((len(t) for t in texts), default=0) + 8)
    ids, n_ids, status = tok.encode_batch(b.text, b.offsets, stride)
    assert (status == 0).all(), status
    bad = [(i, texts[i][:48]) for i in range(len(texts)) if ids[i, :n_ids[i]].tolist() != orc.encode(texts[i]).tolist()]
    assert not bad, bad[:5]


def _word(rnd, n):
    return "".join(rnd.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(n))


def _unit(rnd, c):
    """16 bytes holding exactly c word starts (0 .. 8), the rest spaces."""
    if c == 0:
        return " " * 16
    lens = [1] * c
    for _ in range(16 - 2 * c):       # grow random words while the unit still has room for their spaces
        lens[rnd.randrange(c)] += 1
    s = " ".join(_word(rnd, n) for n in lens)
    return s + " " * (16 - len(s))


def test_units_with_every_count_of_starts(model):
    """Units of 0 .. 8 starts, each repeated over a window and mixed, at every alignment in front of the first; the
    batch packs prompts back to back, so the requests' own alignments vary as well."""
    _, tok, orc = model
    rnd = random.Random(5)
    texts = []
    for off in range(16):
        head = " " * off
        texts.append((head + "a " * 8 * 80).encode())
        texts.append((head + "b" + "a " * 8 * 40).encode())
        for c in range(9):
            texts.append((head + "".join(_unit(rnd, c) for _ in range(40)) + "end").encode())
        texts.append((head + "".join(_unit(rnd, rnd.randint(0, 8)) for _ in range(80))).encode())
    _check(tok, orc, texts)


def test_runs_of_units_without_starts(model):
    """Empty lanes between words: long runs of spaces, and words of 15, 16, 30, 31 and 32 bytes (the last three start
    on byte 1 or 0 of a unit and end on byte 15 of the next), at every alignment."""
    _, tok, orc = model
    rnd = random.Random(7)
    texts = []
    for off in range(16):
        for gap in (17, 33, 100, 300, 511, 530):
            texts.append((" " * off + "a b" + " " * gap + "c d e " + _word(rnd, 5)).encode())
        for n in (15, 16, 30, 31, 32, 47, 48):
            w = _word(rnd, n)
            texts.append((" " * off + "x " + w + " y " + w + " " + " ".join(_word(rnd, 3) for _ in range(70))).encode())
            texts.append(("".join(_unit(rnd, 8) for _ in range(off + 1)) + " " + w + " tail words").encode())
    _check(tok, orc, texts)


def test_63_64_65_complete_words(model):
    """A step takes at most 64 words: with exactly 63, 64 or 65 complete words in the window, and the word after
    them (the 65th's start ends the step) far behind a run of spaces, or cut by the window's end."""
    _, tok, orc = model
    rnd = random.Random(13)
    texts = []
    for n in (63, 64, 65):
        for gap in (1, 2, 15, 16, 17, 40, 200):
            for off in (0, 1, 7, 15):
                words = " ".join(_word(rnd, rnd.randint(1, 3)) for _ in range(n))
                texts.append((" " * off + words + " " * gap + _word(rnd, 4) + " " + _word(rnd, 6)).encode())
                texts.append((" " * off + words + " " * gap + _word(rnd, 40)).encode())
    _check(tok, orc, texts)


def test_words_at_the_window_end(model):
    """Texts whose length puts their end at every offset around a window's last byte, ending inside a word or in a
    space, and words cut by the last byte of a window the text goes on after."""
    _, tok, orc = model
    rnd = random.Random(19)
    texts = []
    for total in range(496, 530):
        for tail in ("", " ", "  "):
            body = " ".join(_word(rnd, rnd.randint(1, 6)) for _ in range(200))
            texts.append((body[:total - len(tail)] + tail).encode())
            texts.append((body[:1024 + total - len(tail)] + tail).encode())
    for cut in range(1, 16):
        for off in range(0, 16, 3):
            pre = " ".join(_word(rnd, 3) for _ in range(130))
            pre = (" " * off + pre)[:511 - cut] + " "
            texts.append((pre + _word(rnd, cut + rnd.randint(0, 10)) + " next words here").encode())
    _check(tok, orc, texts)


def test_step_starting_inside_a_unit(model):
    """A step that starts at byte 1 .. 15 of its first unit, behind the 64th word of the step before, with word starts
    of that unit both in front of the position and behind it."""
    _, tok, orc = model
    rnd = random.Random(29)
    texts = []
    for lead in range(16):
        for after in ("a b", "ab c d", "a", "abcdefg hi"):
            words = " ".join("a" for _ in range(64))            # 64 words in 128 bytes: the step stops at byte 128
            texts.append((" " * lead + words + " " + after + " " + " ".join(_word(rnd, 2) for _ in range(100))).encode())
            texts.append(("b" * (lead + 1) + " " + words + " " + after + " more").encode())
    _check(tok, orc, texts)


def test_random_start_densities_against_express_off(model, oracle):
    """Random per-unit start counts at random alignments and lengths: the express kernel, the buffer-path kernel
    alone (XLLM_SP_EXPRESS=0) and the oracle must agree."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    name, tok, orc = model
    rnd = random.Random(31)
    texts = []
    for _ in range(300):
        units = []
        for _ in range(rnd.randint(1, 120)):
            c = rnd.choice((0, 1, 2, 3, 4, 5, 6, 7, 8, rnd.randint(0, 8)))
            units.append(_unit(rnd, c) if rnd.random() < 0.8 else _word(rnd, rnd.randint(1, 20)) + " ")
        s = " " * rnd.randint(0, 15) + "".join(units)
        texts.append(s[:rnd.randint(1, len(s))].encode())
    want = [orc.encode(t).tolist() for t in texts]
    os.environ["XLLM_SP_EXPRESS"] = "0"
    try:
        h0 = x.Ingest(tokenizer_path=MODELS[name])
    finally:
        del os.environ["XLLM_SP_EXPRESS"]
    try:
        b = workload.pack_prompts(texts)
        stride = 14 * max(len(t) for t in texts) + 8
        for h in (tok, h0):
            ids, n_ids, status = h.encode_batch(b.text, b.offsets, stride)
            assert (status == 0).all()
            bad = [i for i in range(len(texts)) if ids[i, :n_ids[i]].tolist() != want[i]]
            assert not bad, [(i, texts[i][:48]) for i in bad[:5]]
    finally:
        h0.close()
