"""GPU parity of the express tokenizer kernel (csrc/sp_encode.cu: express_run), bit-exact against the CPU oracle, where
a step starts in the middle of a 16-byte unit.  The bytes of that unit in front of the position are left as loaded
(the step before checked them) and only masked out of the word starts; bytes that are not the request's own — in
front of a text that is not 16-byte aligned, or past its end — are rewritten to spaces.  So: requests packed back to
back at every alignment behind foreign bytes of every kind, steps that stop at every offset of a unit behind a word, a
long word, a tab, a line feed or a run of spaces, words against every lane boundary, and texts that end at every offset
of their last window.  Narrow (16-bit ids) and wide kernels, full and truncating rows."""
import os
import random

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
MODELS = {"bpe8k": os.path.join(HERE, "golden", "sp_bpe_8k"), "natural32k": os.path.join(HERE, "golden", "sp_natural_32k")}
HARD = "{}[]{}[]{}[]{}"      # 14 bytes, more ids than a memo payload holds: resolved by the whole warp, then a reload


@pytest.fixture(scope="module", params=[(m, w) for m in MODELS for w in ("narrow", "wide")], ids=lambda p: "-".join(p))
def pair(request, oracle):
    import xllm_service_b200 as x
    model, width = request.param
    old = os.environ.get("XLLM_SP_FORCE_WIDE")
    if width == "wide":
        os.environ["XLLM_SP_FORCE_WIDE"] = "1"      # read when the handle is created
    try:
        h = x.Ingest(tokenizer_path=MODELS[model])
    finally:
        if width == "wide":
            if old is None:
                del os.environ["XLLM_SP_FORCE_WIDE"]
            else:
                os.environ["XLLM_SP_FORCE_WIDE"] = old
    yield h, oracle.SentencePieceOracle(MODELS[model])
    h.close()


def _check(tok, orc, texts, stride=None):
    """Full rows must match the oracle; a row the stride truncates holds the oracle's prefix, with the full count."""
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    if stride is None:
        stride = max(16, 14 * max((len(t) for t in texts), default=0) + 8)
    ids, n_ids, status = tok.encode_batch(b.text, b.offsets, stride)
    bad = []
    for i, t in enumerate(texts):
        want = orc.encode(t).tolist()
        keep = min(len(want), stride)
        if (int(n_ids[i]) != len(want) or int(status[i]) != (1 if len(want) > stride else 0)
                or ids[i, :keep].tolist() != want[:keep]):
            bad.append((i, len(t), int(n_ids[i]), len(want), int(status[i]), t[:48]))
    assert not bad, bad[:5]


def _words(rnd, n, lo=1, hi=9):
    return " ".join("".join(rnd.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(rnd.randint(lo, hi))) for _ in range(n))


def _stop_texts(rnd):
    """Steps that stop at every offset of a unit: behind 64 words, behind a long word, behind a hard word; with a
    space, a tab, a line feed or a run of them just in front of the position."""
    texts = []
    for shift in range(16):
        pad = "p" * shift + " " if shift else ""
        for sep in (" ", "\t", "\n", "    ", " \t ", "\n\n", "\t" * 17, " " * 33):
            tail = _words(rnd, 90, 1, 7)
            texts.append(pad + "a " * 63 + "a" + sep + tail)                   # the 65th word starts the next step
            for long in ("w" * 16, "v" * 17, "u" * 23, "t" * 47, HARD):
                texts.append(pad + long + sep + tail)                           # the position is the long word's end
                texts.append(pad + _words(rnd, 5) + " " + long + sep + "x" + sep + long + sep + tail)
    return [t.encode() for t in texts]


def test_foreign_bytes_in_front_of_a_request(pair):
    """Every alignment 0..15 of a request's first byte, behind a request that ends in a non-ASCII character, in an ASCII
    letter and in a tab; the request starts with short words, with a hard word (whose reload shows the first unit
    again) and with spaces."""
    tok, orc = pair
    rnd = random.Random(41)
    texts, at = [], 0
    for end in ("é", "日", "x", "\t", "\xa0"):
        for first in ("", HARD + " ", "q ", "  ", "z" * 15 + " ", "y" * 16 + " "):
            for a in range(16):
                tail = end.encode()
                body = _words(rnd, rnd.randint(1, 30)).encode() + b" "
                body += b"k" * ((a - at - len(body) - len(tail)) % 16)
                prev = body + tail                                             # ends at a byte offset = a mod 16
                probe = (first + _words(rnd, rnd.randint(1, 120), 1, 7)).encode()
                texts += [prev, probe]
                at += len(prev) + len(probe)
                assert (at - len(probe)) % 16 == a
    _check(tok, orc, texts)


def test_steps_stopping_at_every_offset_of_a_unit(pair):
    tok, orc = pair
    _check(tok, orc, _stop_texts(random.Random(43)))


def test_words_against_lane_boundaries(pair):
    """Words of 1..16 bytes at every offset of a unit (straddling it, ending on its byte 15, starting on its byte 0),
    in the first window and behind a step boundary; one-byte words back to back (8 starts in one lane)."""
    tok, orc = pair
    rnd = random.Random(47)
    texts = []
    for n in range(1, 17):
        for off in range(16):
            w = "".join(rnd.choice("abcdefghijklmnop") for _ in range(n))
            for lead in (off, 496 + off, 1008 + off):
                head = (_words(rnd, lead, 1, 6)[:lead - 1] + " ") if lead else ""
                texts.append(head + w + " " + w + " " + w + "  " + w)
    for shift in range(4):
        texts += [" " * shift + "a " * 300, " " * shift + "a b " * 200 + "cd", "x" * shift + " i" * 270]
    _check(tok, orc, [t.encode() for t in texts])


def test_text_ending_at_every_offset_of_its_last_window(pair):
    tok, orc = pair
    rnd = random.Random(53)
    texts = []
    for size in (40, 560, 1100):
        body = (_words(rnd, 400, 1, 8) + " ").encode()
        texts += [body[:n] for n in range(size - 36, size + 1)]
        texts += [body[:n] + b" " for n in range(size - 20, size)] + [body[:n] + b"\n" for n in range(size - 20, size)]
    _check(tok, orc, texts)


@pytest.mark.parametrize("stride", [1, 40, 333])
def test_truncating_rows(pair, stride):
    tok, orc = pair
    _check(tok, orc, _stop_texts(random.Random(59))[::3], stride=stride)
