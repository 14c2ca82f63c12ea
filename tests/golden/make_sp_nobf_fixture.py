#!/usr/bin/env python3
"""SentencePiece BPE models without byte fallback, and their goldens from upstream libsentencepiece (pip sentencepiece
0.2.1).  Every other BPE fixture was trained with byte_fallback = true, so a char no piece covers comes out as its
<0xNN> byte pieces.  Here it comes out as <unk>, and a run of consecutive unknown symbols comes out as ONE <unk>
(sentencepiece_processor.cc).  That is the "unknown symbol" side of every BPE kernel: sym_ids' unk_id, the lane path's
first / last unknown flags, the cooperative path's merge across its 32-symbol chunks, long_finish's merge in the
long-word pass, and the express kernel's hard-word test and carried unknown flag.

The training corpus is workload sentences with capitals, punctuation, digits and a few non-ASCII letters mixed in.
UNKNOWN_ASCII never occurs in it, so those printable ASCII chars have no piece and reach the ASCII-only express
kernel as unknown symbols.  RARE_CHARS occur a handful of times only, below character_coverage, so they drop out of
the vocabulary too.  main() asserts both.

  nobf_bpe          nmt_nfkc, dummy prefix, split by whitespace, remove_extra_whitespaces (split_mode 1): the express
                    kernel runs, with the word memo and the warm-up kernels.
  nobf_ws_bpe       identity normaliser, kept whitespace, U+2581-run pieces (split_mode 2): words led by U+2581 runs,
                    tab / LF / CR unknown; buffer path only.
  nobf_nodummy_bpe  nmt_nfkc without a dummy prefix (split_mode 1): the first word of a request, and of each text
                    piece of a segmented request, can start with an unknown symbol.
  nobf_nosplit_bpe  trained with split_by_whitespace = false (split_mode 0): pieces span words, a whole text is one
                    pre-token, so texts of more than 512 chars take the long-word pass; identity normaliser with
                    collapsed whitespace.

Outputs (committed):
  tests/golden/sp_<name>/tokenizer.model, tokenizer_config.json     the identity-normaliser models
  tests/golden/sp_<name>.nocharsmap.model                           the nmt_nfkc models without their 240 KB
                                              precompiled charsmap, which is the one sp_bpe_8k's model carries:
                                              materialise() puts it back, and the tests check the result by SHA-256
  tests/golden/sp_nobf_goldens.json   {"sentencepiece_version", "texts": [str], "models": {name: {"split_mode",
                                      "n_pieces", "unk_id", "sha256" of the full model bytes, "ids": [[...] per text]}}}
"texts" (the same for every model) are short adversarial texts, words with unknown runs just past the cooperative path
and a random set over an alphabet rich in unknowns.  seam_texts() (2-16 KB prose, and words past 1 and 2 KB; not frozen)
are checked against the oracle and the wheel at test time, which keeps the committed file small.
Training is single-threaded on a fixed corpus without shuffling, so a run rewrites the same bytes.
Run:  python tests/golden/make_sp_nobf_fixture.py
"""
import hashlib
import io
import json
import os
import random
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from xllm_service_b200 import workload  # noqa: E402

SP = "▁"
TOKENIZER_CONFIG = {"tokenizer_class": "LlamaTokenizer", "add_bos_token": False, "add_eos_token": False}
NAMES = ["nobf_bpe", "nobf_ws_bpe", "nobf_nodummy_bpe", "nobf_nosplit_bpe"]
NFKC = ("nobf_bpe", "nobf_nodummy_bpe")          # committed without the charsmap (see the module docstring)
# the layout each model must have, as the loader reports it (xllm_tokenizer_probe)
LAYOUT = {
    "nobf_bpe": {"split_mode": 1, "byte_fallback": 0},
    "nobf_ws_bpe": {"split_mode": 2, "trie_units": 0, "byte_fallback": 0},
    "nobf_nodummy_bpe": {"split_mode": 1, "byte_fallback": 0},
    "nobf_nosplit_bpe": {"split_mode": 0, "byte_fallback": 0},
}
UNKNOWN_ASCII = "`~^|{}\\7"           # never in the corpus: no piece
RARE_CHARS = "ø語ʃж"                   # a few times in the corpus: below character_coverage
COMMON_CHARS = "éü日本ß"               # often enough to be pieces
PUNCT = ".,;:!?()[]<>\"'=+-*/_#$%&@"
DIGITS = "012345689"                 # every digit but 7
COVERAGE = 0.9995


def model_dir(name, golden_dir=HERE):
    return os.path.join(golden_dir, "sp_" + name)


def _normalizer_edit(blob, edit):
    """blob with its NormalizerSpec (ModelProto field 3) replaced by edit(spec bytes); every other record verbatim."""
    sys.path.insert(0, HERE)
    import make_wide_fixtures as mw
    out = bytearray()
    for num, wt, val, raw in mw._fields(blob):
        if num == 3:
            spec = edit(bytes(val))
            raw = b"\x1a" + mw._put_varint(len(spec)) + spec
        out += raw
    return bytes(out)


def _spec_records(spec):
    sys.path.insert(0, HERE)
    import make_wide_fixtures as mw
    return [(num, bytes(raw)) for num, wt, val, raw in mw._fields(spec)]


def strip_charsmap(blob):
    """The model without NormalizerSpec.precompiled_charsmap (field 2)."""
    return _normalizer_edit(blob, lambda spec: b"".join(r for n, r in _spec_records(spec) if n != 2))


def nfkc_charsmap_record(golden_dir=HERE):
    """The nmt_nfkc precompiled_charsmap record of the committed sp_bpe_8k model."""
    sys.path.insert(0, HERE)
    import make_wide_fixtures as mw
    with open(os.path.join(golden_dir, "sp_bpe_8k", "tokenizer.model"), "rb") as f:
        base = f.read()
    spec = next(bytes(val) for num, wt, val, raw in mw._fields(base) if num == 3)
    return next(r for n, r in _spec_records(spec) if n == 2)


def restore_charsmap(stripped, golden_dir=HERE):
    """The full model: the charsmap record back right after the normaliser's name (field 1), where protobuf writes it."""
    cm = nfkc_charsmap_record(golden_dir)
    return _normalizer_edit(stripped, lambda spec: b"".join(r + (cm if n == 1 else b"") for n, r in _spec_records(spec)))


def materialise(name, root, golden_dir=HERE):
    """The directory of one model: the committed one, or (NFKC) a fresh one under root with the full model."""
    if name not in NFKC:
        return model_dir(name, golden_dir)
    d = os.path.join(str(root), "sp_" + name)
    os.makedirs(d, exist_ok=True)
    with open(model_dir(name, golden_dir) + ".nocharsmap.model", "rb") as f:
        blob = restore_charsmap(f.read(), golden_dir)
    with open(os.path.join(d, "tokenizer.model"), "wb") as f:
        f.write(blob)
    with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
        json.dump(TOKENIZER_CONFIG, f)
    return d


# ---------------------------------------------------------------------------- training corpus
def corpus(seed, n=12000, kept_ws=False):
    """workload sentences with capitals, punctuation, digits (no 7) and common non-ASCII letters mixed in, and each
    rare char a few times.  kept_ws: indentation and doubled spaces too (the identity-normaliser model learns U+2581-run
    pieces from them); no tab / LF / CR, which stay unknown."""
    rnd = random.Random(seed)
    out = []
    for s in workload.sentences(n, (3, 30), seed=seed):
        words = []
        for w in s.split(" "):
            r = rnd.random()
            if r < 0.12:
                w = w.capitalize()
            elif r < 0.15:
                w = w.upper()
            r = rnd.random()
            if r < 0.10:
                w += rnd.choice(".,;:!?")
            elif r < 0.14:
                a, b = rnd.choice(("()", "[]", "<>", '""', "''"))
                w = a + w + b
            elif r < 0.17:
                w = "".join(rnd.choice(DIGITS) for _ in range(rnd.randint(1, 6)))
            elif r < 0.25:
                w = w + rnd.choice("=+-*/_#$%&@") + rnd.choice((w, "x", "1"))
            elif r < 0.28:
                c = rnd.choice(COMMON_CHARS)
                i = rnd.randrange(len(w) + 1)
                w = w[:i] + c + w[i:]
            words.append(w)
        if kept_ws:
            r = rnd.random()
            if r < 0.3:
                out.append(" " * rnd.choice((2, 4, 4, 8)) + " ".join(words))
                continue
            if r < 0.5:
                out.append("  ".join(words))
                continue
        out.append(" ".join(words))
    for i, c in enumerate(RARE_CHARS):   # each rare char a few times, far below 1 - COVERAGE of the corpus
        for k in range(3):
            out[(i * 997 + k * 131) % len(out)] += " " + c + "x"
    text = "".join(out)
    assert not set(UNKNOWN_ASCII) & set(text)
    return out


def train(name):
    import sentencepiece as spm
    common = dict(num_threads=1, input_sentence_size=0, shuffle_input_sentence=False, minloglevel=2,
                  character_coverage=COVERAGE, byte_fallback=False, model_type="bpe")
    model = io.BytesIO()
    if name == "nobf_bpe":
        spm.SentencePieceTrainer.train(sentence_iterator=iter(corpus(501)), model_writer=model, vocab_size=3000,
                                       **common)
    elif name == "nobf_ws_bpe":
        spm.SentencePieceTrainer.train(
            sentence_iterator=iter(corpus(502, kept_ws=True)), model_writer=model, vocab_size=3000,
            normalization_rule_name="identity", remove_extra_whitespaces=False, allow_whitespace_only_pieces=True,
            **common)
    elif name == "nobf_nodummy_bpe":
        spm.SentencePieceTrainer.train(sentence_iterator=iter(corpus(503)), model_writer=model, vocab_size=3000,
                                       add_dummy_prefix=False, **common)
    elif name == "nobf_nosplit_bpe":
        spm.SentencePieceTrainer.train(sentence_iterator=iter(corpus(504, n=10000)), model_writer=model,
                                       vocab_size=3000, split_by_whitespace=False,
                                       normalization_rule_name="identity", **common)
    else:
        raise ValueError(name)
    return model.getvalue()


# ---------------------------------------------------------------------------- layout checks
def check_model(name, blob, d):
    """Asserts the model (bytes blob, written in directory d) has the layout and the unknown chars it was built for:
    from the proto, through the wheel, and through the loader when the library is built."""
    import sentencepiece as spm
    from sentencepiece import sentencepiece_model_pb2 as pb
    m = pb.ModelProto()
    m.ParseFromString(blob)
    assert m.trainer_spec.model_type == pb.TrainerSpec.BPE and not m.trainer_spec.byte_fallback, name
    n = m.normalizer_spec
    assert (n.name == "identity") == (name in ("nobf_ws_bpe", "nobf_nosplit_bpe")), name
    assert n.remove_extra_whitespaces == (name != "nobf_ws_bpe"), name
    assert n.add_dummy_prefix == (name != "nobf_nodummy_bpe"), name
    assert m.trainer_spec.split_by_whitespace == (name != "nobf_nosplit_bpe"), name
    sp = spm.SentencePieceProcessor(model_proto=blob)
    unk = sp.unk_id()
    for c in UNKNOWN_ASCII + RARE_CHARS:
        assert sp.PieceToId(c) == unk, (name, c)
        assert unk in sp.EncodeAsIds("ab" + c + "cd"), (name, c)
    for c in COMMON_CHARS + PUNCT + DIGITS + "abcxyzABCXYZ":
        assert sp.PieceToId(c) != unk, (name, c)
    if name == "nobf_ws_bpe":
        assert sp.PieceToId(SP * 4) != unk
        for c in "\t\n\r":
            assert sp.PieceToId(c) == unk, (name, repr(c))
    try:
        from xllm_service_b200 import _lib
        info = _lib.tokenizer_probe(d)
    except Exception as e:  # noqa: BLE001  the library is not built: the checks above stand alone
        if "not built" not in str(e):
            raise
        return
    for k, v in LAYOUT[name].items():
        assert info[k] == v, (name, k, info[k], v)
    assert info["unk_id"] == unk and info["n_pieces"] == sp.GetPieceSize(), name


# ---------------------------------------------------------------------------- golden texts
def letters(rnd, n, alphabet="abcdefghijklmnopqrstuvwxyz"):
    return "".join(rnd.choice(alphabet) for _ in range(n))


def unk_run(rnd, n):
    return "".join(rnd.choice(UNKNOWN_ASCII) for _ in range(n))


def words_text(rnd, nbytes, alphabet="abcdefghijklmnopqrstuvwxyz"):
    out, size = [], 0
    while size < nbytes:
        w = letters(rnd, rnd.randint(1, 9), alphabet)
        out.append(w)
        size += len(w) + 1
    return " ".join(out)[:nbytes]


def word_with_unknowns(rnd, nbytes, run=None):
    """A word of nbytes ASCII bytes (no space) holding unknown runs: one run of `run` unknowns at a random place, or
    several short ones."""
    if run is not None:
        run = min(run, nbytes)
        a = rnd.randint(0, nbytes - run)
        return letters(rnd, a) + unk_run(rnd, run) + letters(rnd, nbytes - run - a)
    out = []
    while len(out) < nbytes:
        out += list(unk_run(rnd, rnd.randint(1, 4)) if rnd.random() < 0.3 else letters(rnd, rnd.randint(1, 5)))
    return "".join(out[:nbytes])


def adversarial_texts(rnd):
    """Short texts at the unknown-symbol seams (frozen as goldens)."""
    t = ["", " ", "|", "||", " | ", "7", "77", "a7b", "x 7 y", "7 7", "~`^|{}\\7", "a|b", "|ab", "ab|", "|a|", "a||b",
         "|| ab ||", "ab| |cd", "ab|  |cd", "ab|\t|cd", "ab|\n|cd", "ab|\r\n|cd", "ab|" + SP + "|cd",
         "ab| " + SP + " |cd", "|" + SP + "|", SP + "|", "|" + SP, "| | | |", "|  |  |", "|\t|\n|",
         "ab|é", "|é", "ab ~é cd", "x|日本 y", "|ø", "ø|", "øø|ø", "7語", "語語語 x", "a ж b", "ʃʃ|ʃ",
         "日本語テキスト", "テキスト|", "\U0001F600\U0001F600\U0001F600", "ab\U0001F600|cd", "|\U0001F600|",
         "Hello, World! (x+1)*2 = 42; {key: value} ~user/path | grep `cmd` ^ 7",
         "if (a[7] != b) { return c ^ d; } // ~7",
         "  leading spaces |", "trailing |  ", "\t|tab lead", "|\n", "a　|　b", "ﬁ|ﬁ", "Ａ|Ｂ", "①|②"]
    for k in range(1, 41):
        r = unk_run(rnd, k)
        t.append("a " + r + " b")
        if k in (1, 2, 3, 15, 16, 17, 32, 33, 40):
            t += [r, "ab" + r + "cd", r + "x", "x" + r]
    for pos in ("start", "middle", "end"):
        for n in (2, 5, 9, 14):
            w = letters(rnd, n)
            u = unk_run(rnd, rnd.randint(1, 3))
            word = u + w if pos == "start" else (w + u if pos == "end" else w[:n // 2] + u + w[n // 2:])
            t += [word, "one " + word + " " + word]
    for n in (14, 15, 16, 17, 18):                    # the express lane path takes words of up to 15 bytes
        for run in (1, 3, n):
            w = word_with_unknowns(rnd, n, run)
            t += [w, "head " + w + " tail " + w]
    for n in (32, 33, 34):                            # the buffer path's lane columns hold 32 symbols
        t.append("x " + word_with_unknowns(rnd, n, rnd.randint(1, n)) + " y")
    for run, n in ((33, 33), (33, 50), (40, 200), (64, 64), (65, 90), (70, 512)):   # across the 32-symbol chunks
        t.append("w " + word_with_unknowns(rnd, n, run) + " z")
    for n in (40, 300):
        t.append(word_with_unknowns(rnd, n) + " " + word_with_unknowns(rnd, n))
    return [s.encode() for s in t]


def long_word_texts(rnd, sizes):
    """Unknown runs inside words past the cooperative path (512 chars) and past the 2 KB normalised-text buffer."""
    return [("start " + word_with_unknowns(rnd, n, run) + " end").encode() for n, run in sizes]


RANDOM_ALPHABET = list("abcdefgxyz") + list(UNKNOWN_ASCII) * 2 + [
    " ", " ", "  ", "\t", "\n", SP, "é", "日本", "ø", "語", "\U0001F600", "Ab", "42", ".", "||", "~~~", "0"]


def random_texts(rnd, n=300, most=80):
    return ["".join(rnd.choice(RANDOM_ALPHABET) for _ in range(rnd.randrange(0, most))).encode() for _ in range(n)]


def golden_texts():
    """The texts frozen in sp_nobf_goldens.json "texts"."""
    rnd = random.Random(2581)
    return (adversarial_texts(rnd) + long_word_texts(rnd, ((513, 33), (530, 40))) + [b"a" * 510 + b"||" + b"b" * 30]
            + random_texts(rnd, 50))


def prose_with_unknowns(rnd, size):
    """About size bytes of short words with unknown-holding words of 1-15, 16-120 and 500-600 bytes sprinkled in."""
    parts, n = [], 0
    while n < size:
        r = rnd.random()
        if r < 0.75:
            p = letters(rnd, rnd.randint(1, 9))
        elif r < 0.9:
            p = word_with_unknowns(rnd, rnd.randint(1, 15))
        elif r < 0.97:
            p = word_with_unknowns(rnd, rnd.randint(16, 120), rnd.choice((None, 33, 40)))
        else:
            p = word_with_unknowns(rnd, rnd.randint(500, 600))
        parts.append(p)
        n += len(p) + 1
    return " ".join(parts).encode()


def seam_texts():
    """Longer texts, not frozen: prose of 2-16 KB (one with a non-ASCII char late in it, an express hand-over) and
    unknown runs in words past 512 and 2048 bytes."""
    rnd = random.Random(11)
    out = [prose_with_unknowns(rnd, size) for size in (2000, 5000, 9000, 16000)]
    out[2] = out[2][:7000] + " ab|é cd ".encode() + out[2][7000:]
    out += long_word_texts(rnd, ((600, 40), (700, 65), (1025, 70), (1100, 40), (2100, 64), (2100, 40)))
    out.append(word_with_unknowns(rnd, 1500).encode())
    return out


def main():
    import sentencepiece as spm
    texts = golden_texts()
    out = {"sentencepiece_version": spm.__version__, "texts": [t.decode() for t in texts], "models": {}}
    for name in NAMES:
        blob = train(name)
        if name in NFKC:
            stripped = strip_charsmap(blob)
            assert restore_charsmap(stripped) == blob, name     # the charsmap is sp_bpe_8k's, byte for byte
            with open(model_dir(name) + ".nocharsmap.model", "wb") as f:
                f.write(stripped)
            d = materialise(name, tempfile.mkdtemp())          # checked here, never committed
        else:
            d = model_dir(name)
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, "tokenizer.model"), "wb") as f:
                f.write(blob)
            with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
                json.dump(TOKENIZER_CONFIG, f)
        check_model(name, blob, d)
        sp = spm.SentencePieceProcessor(model_proto=blob)
        ids = [sp.EncodeAsIds(t) for t in texts]
        out["models"][name] = {"split_mode": LAYOUT[name]["split_mode"], "n_pieces": sp.GetPieceSize(),
                               "unk_id": sp.unk_id(), "sha256": hashlib.sha256(blob).hexdigest(), "ids": ids}
        n_unk = sum(x.count(sp.unk_id()) for x in ids)
        print("%-17s %7d bytes  %5d pieces  %4d texts  %5d <unk>" % (name, len(blob), sp.GetPieceSize(), len(ids),
                                                                      n_unk))
    with open(os.path.join(HERE, "sp_nobf_goldens.json"), "w", encoding="utf-8") as f:
        json.dump(out, f, separators=(",", ":"), ensure_ascii=False)


if __name__ == "__main__":
    main()
