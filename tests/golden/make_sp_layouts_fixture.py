#!/usr/bin/env python3
"""SentencePiece models in the layouts the other fixtures do not have, and their goldens from upstream
libsentencepiece (pip sentencepiece 0.2.1).  Every other SentencePiece fixture is nmt_nfkc with collapsed whitespace, a
dummy prefix, no piece holding U+2581 past its first char, pieces of at most 18 bytes and at most 5 Unigram pieces
starting at one position.  These five are not:

  llama_bpe      BPE, identity normaliser, kept whitespace, U+2581-run pieces (split_mode 2), byte fallback, split
                 digits: the Llama-2 / Mistral tokenizer.model layout.  No piece for tab / CR / LF / NUL, so those come
                 out as <0xNN> byte pieces.
  nodummy_bpe    nmt_nfkc BPE with add_dummy_prefix = false (split_mode 1, express kernel eligible).
  ws_unigram     Unigram, identity normaliser, kept whitespace, U+2581-run pieces (split_mode 2), byte fallback.
  nosplit_bpe    BPE trained with split_by_whitespace = false: pieces that span words ("▁of▁the", split_mode 0);
                 identity normaliser with collapsed whitespace.
  chain_unigram  a hand-built Unigram ModelProto (normaliser of sp_unigram_4k): a..z, the chains a^k (k = 2..64),
                 "▁" + b^k (up to 64 bytes) and the prefixes of (0123456789)^7 (lengths 2..64), so more than 32 pieces
                 start at one position and pieces of 31, 32 and 33 bytes start at the same one.  Scores are multiples of
                 1/4, so float32 path sums are exact and many competing paths tie exactly.

Outputs (committed):
  tests/golden/sp_layout_<name>/tokenizer.model, tokenizer_config.json   (all but chain_unigram, which the tests
                                              rebuild with chain_unigram() / materialise())
  tests/golden/sp_layouts_goldens.json        {"sentencepiece_version", "models": {name: {"split_mode", "n_pieces",
                                              "sha256" of the model bytes, "cases": [{"text": hex, "ids": [...]}]}}}
The goldens hold short texts; the long seam texts (seam_texts()) are deterministic and checked against the oracle and
the wheel at test time, which keeps the committed file small.
Training is single-threaded on a fixed corpus without shuffling, so a run rewrites the same bytes.
Run:  python tests/golden/make_sp_layouts_fixture.py
"""
import hashlib
import io
import json
import os
import random
import struct
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from xllm_service_b200 import workload  # noqa: E402

SP = "▁"
TOKENIZER_CONFIG = {"tokenizer_class": "LlamaTokenizer", "add_bos_token": False, "add_eos_token": False}
NAMES = ["llama_bpe", "nodummy_bpe", "ws_unigram", "nosplit_bpe", "chain_unigram"]
# the layout each model must have: split_mode as the loader computes it (sp_model.cc), and normaliser flags
LAYOUT = {
    "llama_bpe": {"split_mode": 2, "trie_units": 0, "byte_fallback": 1},
    "nodummy_bpe": {"split_mode": 1, "byte_fallback": 1},
    "ws_unigram": {"split_mode": 2, "trie_units": 0, "byte_fallback": 1},
    "nosplit_bpe": {"split_mode": 0},
    "chain_unigram": {"split_mode": 1},
}


def model_dir(name, golden_dir=HERE):
    return os.path.join(golden_dir, "sp_layout_" + name)


# ---------------------------------------------------------------------------- training corpora
def ws_corpus(seed, n=12000):
    """workload sentences with indentation, doubled spaces and line breaks mixed in (identity-normaliser models learn
    U+2581-run pieces from it), and a few digit runs.  A broken sentence goes in as one indented line per sentence, as
    Llama's corpus did: a newline inside a sentence would become a piece of its own, and the layout wants LF to come
    out as the byte piece <0x0A>."""
    rnd = random.Random(seed)
    out = []
    for s in workload.sentences(n, (3, 30), seed=seed):
        words = s.split(" ")
        r = rnd.random()
        if r < 0.3:
            out.append(" " * rnd.choice((2, 4, 4, 8, 8, 12)) + s)
        elif r < 0.5:
            out += [" " * rnd.choice((0, 4, 8)) + " ".join(words[i:i + 4]) for i in range(0, len(words), 4)]
        elif r < 0.7:
            out.append("  ".join(words))
        elif r < 0.8:
            out.append(s + " " + str(rnd.randrange(10 ** 6)))
        else:
            out.append(s)
    return out


def train(name):
    import sentencepiece as spm
    common = dict(num_threads=1, input_sentence_size=0, shuffle_input_sentence=False, minloglevel=2,
                  character_coverage=1.0)
    model = io.BytesIO()
    if name == "llama_bpe":
        spm.SentencePieceTrainer.train(
            sentence_iterator=iter(ws_corpus(101)), model_writer=model, model_type="bpe", vocab_size=4000,
            normalization_rule_name="identity", remove_extra_whitespaces=False, add_dummy_prefix=True,
            allow_whitespace_only_pieces=True, split_digits=True, byte_fallback=True, **common)
    elif name == "nodummy_bpe":
        spm.SentencePieceTrainer.train(
            sentence_iterator=iter(workload.sentences(12000, seed=202)), model_writer=model, model_type="bpe",
            vocab_size=3000, add_dummy_prefix=False, byte_fallback=True, **common)
    elif name == "ws_unigram":
        spm.SentencePieceTrainer.train(
            sentence_iterator=iter(ws_corpus(303)), model_writer=model, model_type="unigram", vocab_size=3000,
            normalization_rule_name="identity", remove_extra_whitespaces=False, allow_whitespace_only_pieces=True,
            byte_fallback=True, **common)
    elif name == "nosplit_bpe":
        spm.SentencePieceTrainer.train(
            sentence_iterator=iter(workload.sentences(12000, (3, 12), seed=404)), model_writer=model,
            model_type="bpe", vocab_size=3000, split_by_whitespace=False, normalization_rule_name="identity", **common)
    else:
        raise ValueError(name)
    return model.getvalue()


def chain_unigram(golden_dir=HERE):
    """The hand-built chain model (see the module docstring) as ModelProto bytes: the pieces below, then every other
    record of sp_unigram_4k's model verbatim (its normaliser spec with the nmt_nfkc charsmap, and its trainer spec with
    vocab_size set to the piece count).  Pure Python and deterministic, so the tests rebuild it from the committed
    sp_unigram_4k model instead of committing a second copy of the 240 KB charsmap."""
    sys.path.insert(0, HERE)
    import make_wide_fixtures as mw
    with open(os.path.join(golden_dir, "sp_unigram_4k", "tokenizer.model"), "rb") as f:
        base = f.read()
    rnd = random.Random(64)
    pieces = [("<unk>", 0.0, 2), ("<s>", 0.0, 3), ("</s>", 0.0, 3)]   # UNKNOWN, CONTROL (NORMAL = 1)
    normal = [(SP, -2.0)] + [(chr(c), -3.0 - (c % 5) * 0.25) for c in range(ord("a"), ord("z") + 1)]
    normal += [(str(d), -3.0) for d in range(10)]
    # chain score: -(bytes) * 2.5 plus a bonus in quarter steps, so long and short pieces both win somewhere
    bonus = lambda: rnd.choice((0.0, 0.25, 0.5, 1.0, 1.5, 2.0, 2.5, 3.0))  # noqa: E731
    normal += [("a" * k, -2.5 * k + bonus()) for k in range(2, 65)]
    normal += [(SP + "b" * k, -2.5 * (k + 1) + bonus()) for k in range(1, 62)]
    digits = "0123456789" * 7
    normal += [(digits[:k], -2.5 * k + bonus()) for k in range(2, 65)]
    pieces += [(p, sc, 1) for p, sc in normal]
    out = bytearray()
    for p, sc, typ in pieces:   # ModelProto.SentencePiece {1: piece, 2: score, 3: type}
        pb = p.encode()
        body = b"\x0a" + mw._put_varint(len(pb)) + pb + b"\x15" + struct.pack("<f", sc) + b"\x18" + mw._put_varint(typ)
        out += b"\x0a" + mw._put_varint(len(body)) + body
    for num, wt, val, raw in mw._fields(base):
        if num == 1:
            continue
        if num == 2:            # TrainerSpec: vocab_size (field 4) = the piece count
            ts = bytearray()
            for n2, w2, v2, r2 in mw._fields(bytes(val)):
                ts += (b"\x20" + mw._put_varint(len(pieces))) if n2 == 4 else r2
            raw = b"\x12" + mw._put_varint(len(ts)) + bytes(ts)
        out += raw
    return bytes(out)


def materialise(name, root, golden_dir=HERE):
    """The directory of one model: the committed one, or (chain_unigram) a fresh one under root built by
    chain_unigram()."""
    if name != "chain_unigram":
        return model_dir(name, golden_dir)
    d = os.path.join(str(root), "sp_layout_chain_unigram")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "tokenizer.model"), "wb") as f:
        f.write(chain_unigram(golden_dir))
    with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
        json.dump(TOKENIZER_CONFIG, f)
    return d


# ---------------------------------------------------------------------------- layout checks
def proto_layout(blob):
    """split_mode from the model's pieces (the loader's rule, sp_model.cc), and the normaliser flags."""
    from sentencepiece import sentencepiece_model_pb2 as pb
    m = pb.ModelProto()
    m.ParseFromString(blob)
    inside, only_after = False, True
    for p in m.pieces:
        if p.type != pb.ModelProto.SentencePiece.NORMAL:
            continue
        for c in range(1, len(p.piece)):
            if p.piece[c] == SP:
                inside = True
                only_after &= p.piece[c - 1] == SP
    n = m.normalizer_spec
    return {"split_mode": 1 if not inside else (2 if only_after else 0), "name": n.name,
            "add_dummy_prefix": n.add_dummy_prefix, "remove_extra_whitespaces": n.remove_extra_whitespaces,
            "max_piece_len": max(len(p.piece.encode()) for p in m.pieces), "pieces": [p.piece for p in m.pieces]}


def check_layout(name, blob, d):
    """Asserts the model (bytes blob, written in directory d) has the layout it was built for: through the loader when
    the library is built, and always from the proto itself."""
    lay = proto_layout(blob)
    want = LAYOUT[name]
    assert lay["split_mode"] == want["split_mode"], (name, lay["split_mode"])
    kept_ws = name in ("llama_bpe", "ws_unigram")
    assert (lay["name"] == "identity") == (kept_ws or name == "nosplit_bpe"), name
    assert lay["remove_extra_whitespaces"] == (not kept_ws), name
    assert lay["add_dummy_prefix"] == (name != "nodummy_bpe"), name
    if lay["split_mode"] == 2:
        assert {SP * 4, SP * 8} <= set(lay["pieces"]), name
        assert not {"\n", "\t", "\r"} & set(lay["pieces"]), name
    if name == "nosplit_bpe":
        assert sum(SP in p[1:] for p in lay["pieces"]) >= 100, "no cross-word pieces"
    if name == "chain_unigram":
        assert lay["max_piece_len"] == 64
    try:
        from xllm_service_b200 import _lib
        info = _lib.tokenizer_probe(d)
    except Exception as e:  # noqa: BLE001  the library is not built: the proto check above stands alone
        if "not built" not in str(e):
            raise
        return lay
    for k, v in want.items():
        assert info[k] == v, (name, k, info[k], v)
    return lay


# ---------------------------------------------------------------------------- golden texts
def words_text(rnd, nbytes, alphabet="abcdefghijklmnopqrstuvwxyz"):
    out, size = [], 0
    while size < nbytes:
        w = "".join(rnd.choice(alphabet) for _ in range(rnd.randint(1, 9)))
        out.append(w)
        size += len(w) + 1
    return " ".join(out)[:nbytes]


def code_text(rnd, lines):
    """Python-like code with 4-, 8- and 12-space indentation."""
    out = []
    for i in range(lines):
        ind = " " * rnd.choice((0, 4, 8, 12))
        out.append(ind + rnd.choice(("def f%d(x, y):" % i, "return x + %d" % i, "if x  ==  y:", "for i in range(10):",
                                     "print('hello  world')", "# a comment", "", "x = [1, 2, 3]")))
    return "\n".join(out)


def chat_text(rnd, most):
    msgs = []
    for role in ("system", "user", "assistant", "user"):
        msgs.append("<|%s|>\n%s\n" % (role, words_text(rnd, rnd.randint(5, most))))
    return "".join(msgs) + "<|assistant|>\n"


def ws_texts(rnd):
    """Short texts aimed at the whitespace seams of the identity / kept-whitespace layouts (frozen as goldens)."""
    t = ["", " ", "  ", "a", " a", "a ", "  a  b  ", "hello world", "hello  world", "\thello\tworld\t",
         "line one\nline two\r\nline three\r", "\n", "\n\n\n", "\r\n", "a\x00b", "\x00", " \x00 ", "\x00\x00 x",
         SP, SP + " " + SP, " " + SP + " ", "a " + SP + SP + " b", SP * 3 + "  x", "x  " + SP, "café  naïve",
         "日本語  テキスト", "tab\t\tx", "1234567890  42", "  ends with spaces    ",
         "    leading four", "\n    indented after newline", "ﬁne  ①  ｆｕｌｌ"]
    for k in (1, 2, 3, 4, 5, 7, 8, 9, 12, 13, 16, 17, 31, 32, 33, 40, 169, 170, 171, 172, 175, 600):
        t.append("x" + " " * k + "y")
        if k in (1, 2, 4, 8, 33, 170, 171, 600):
            t += [" " * k + "lead", "trail" + " " * k, " " * k]
    for _ in range(4):
        t.append(code_text(rnd, rnd.randint(3, 12)))
    t.append(chat_text(rnd, 60))
    out = [s.encode() for s in t]
    out += [b"\xff\xfe  invalid \x80\x81", b"trunc \xe6\x97  ", b"  \xc0\xaf overlong", b"ok\xe2\x96\x81\xe2",
            b"\xe2\x96\x81 \xe2\x96\x81\xe2\x96", b"\x00\xff  \n"]
    alphabet = list("abcdefghij      \t\n\r") + ["\x00", SP, "é", "日", "\U0001F600", "  ", "    ", "0", "7"]
    for _ in range(50):
        out.append("".join(rnd.choice(alphabet) for _ in range(rnd.randrange(1, 60))).encode())
    for _ in range(12):
        out.append(bytes(rnd.getrandbits(8) for _ in range(rnd.randrange(1, 30))))
    out += [s.encode() for s in workload.sentences(12, (1, 20), seed=rnd.randrange(1 << 30))]
    return out


def nodummy_texts(rnd):
    """No dummy prefix: text that starts with and without a space, and a non-ASCII char mid-prompt (an express
    hand-over)."""
    out = ws_texts(rnd)
    for _ in range(16):
        out.append(handover_text(rnd, rnd.randint(0, 120), rnd.randint(0, 60)).encode())
    return out


def handover_text(rnd, head, tail):
    odd = ["été", "日本", "\U0001F600", "ＡＢ", "①", "naïve", " "]
    return (rnd.choice(("", " ", "  ", "\t")) + words_text(rnd, head) + rnd.choice((" ", "", "  ")) + rnd.choice(odd) +
            rnd.choice((" ", "")) + words_text(rnd, tail))


def chain_texts(rnd, n_mixed=16):
    t = []
    for k in (1, 2, 3, 30, 31, 32, 33, 34, 40, 63, 64, 65, 66, 100, 200):
        t += ["a" * k, "b" * k, "0123456789" * (k // 10) + "0123456789"[:k % 10]]
    t += ["b" * 40 + "a" * 40, "c" * 35 + "a" * 40, "xy" + "a" * 33 + "z" + "a" * 70, "c" * 40 + "0123456789" * 5,
          "b" * 31 + "a" * 31 + "b" * 33, "ab" * 40]
    for _ in range(n_mixed):
        parts = []
        for _ in range(rnd.randint(1, 8)):
            c = rnd.random()
            if c < 0.3:
                parts.append("a" * rnd.randint(1, 120))
            elif c < 0.5:
                parts.append("b" * rnd.randint(1, 70))
            elif c < 0.65:
                parts.append(("0123456789" * 8)[:rnd.randint(1, 75)])
            else:
                parts.append(words_text(rnd, rnd.randint(1, 30)))
        t.append(rnd.choice((" ", "")).join(parts))
    t += ["hello " + "a" * 40 + " world " + "b" * 33 + " 0123456789012345678901234567890123 x", "é" + "a" * 40]
    return [s.encode() for s in t]


def golden_texts(name):
    """The texts frozen in sp_layouts_goldens.json: short ones, so the file stays small; the long seam texts are
    seam_texts() and are checked against the oracle (and the wheel, when it imports) live."""
    rnd = random.Random(sum(map(ord, name)))
    if name == "nodummy_bpe":
        return nodummy_texts(rnd)
    if name == "nosplit_bpe":
        return ws_texts(rnd) + [s.encode() for s in workload.sentences(6, (40, 120), seed=rnd.randrange(1 << 30))]
    if name == "chain_unigram":
        return chain_texts(rnd)
    return ws_texts(rnd)


def seam_texts(name):
    """Long texts at the kernels' seams, deterministic but not frozen: space runs that straddle byte 127 / 128 of a
    128-byte fast window and the 512-byte express window, runs that straddle the 2 KB normalized-text drain point,
    runs longer than the 1 KB long-word threshold, indented code and chat-like prompts, express hand-overs deep into a
    prompt (nodummy_bpe), whole prompts of 5-20 KB as one pre-token (nosplit_bpe), chains inside text
    (chain_unigram)."""
    rnd = random.Random(7 + sum(map(ord, name)))
    if name == "chain_unigram":
        return chain_texts(rnd, 60)
    t = []
    for win in (128, 512):
        for start in range(win - 6, win + 2):
            for run in (1, 2, 3, 5, 9):
                t.append(words_text(rnd, start).ljust(start, "q") + " " * run + words_text(rnd, 40))
    for start in (650, 670, 680, 682, 684, 690, 2030, 2040, 2046, 2048):
        t.append(words_text(rnd, start) + " " * rnd.choice((3, 7, 20, 60)) + words_text(rnd, 300))
    for run in (342, 345, 400, 700, 1100):
        t.append(words_text(rnd, 100) + " " * run + "word" + " " * 3 + words_text(rnd, 100))
    t += [code_text(rnd, rnd.randint(20, 80)) for _ in range(8)]
    t += [chat_text(rnd, 200) for _ in range(6)]
    if name == "nodummy_bpe":
        t += [handover_text(rnd, rnd.randint(0, 1500), rnd.randint(0, 1500)) for _ in range(60)]
    out = [s.encode() for s in t]
    if name == "nosplit_bpe":
        out += [" ".join(workload.sentences(n // 60, (8, 12), seed=n)).encode()[:n] for n in (5000, 9000, 14000, 20000)]
    return out


def main():
    import sentencepiece as spm
    out = {"sentencepiece_version": spm.__version__, "models": {}}
    for name in NAMES:
        if name == "chain_unigram":
            blob = chain_unigram()
            d = materialise(name, tempfile.mkdtemp())   # checked here, never committed
        else:
            blob = train(name)
            d = model_dir(name)
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, "tokenizer.model"), "wb") as f:
                f.write(blob)
            with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
                json.dump(TOKENIZER_CONFIG, f)
        check_layout(name, blob, d)
        sp = spm.SentencePieceProcessor(model_proto=blob)
        cases = [{"text": t.hex(), "ids": sp.EncodeAsIds(t)} for t in golden_texts(name)]
        out["models"][name] = {"split_mode": LAYOUT[name]["split_mode"], "n_pieces": sp.GetPieceSize(),
                               "sha256": hashlib.sha256(blob).hexdigest(), "cases": cases}
        print("%-14s %7d bytes  %5d pieces  %4d cases" % (name, len(blob), sp.GetPieceSize(), len(cases)))
    with open(os.path.join(HERE, "sp_layouts_goldens.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
