#!/usr/bin/env python3
"""Large-id tokenizer models derived from the committed small ones, and their goldens.

A derived model is a committed model with N filler pieces spliced in front of its first NORMAL piece (SentencePiece) or
its first merge (tiktoken).  No text can ever produce a filler:
  SentencePiece  a filler is two supplementary private-use chars (U+F0000..), which no test text holds and which are
                 not pieces on their own; filler scores lie between the real NORMAL scores, interleaved evenly, so a
                 BPE model's real merges get ranks past 65 535 as well and a Unigram model keeps its min / max score
                 (its unknown-char score, min_score - 10, is unchanged)
  tiktoken       a filler is a 3-byte token starting with 0xF8..0xFF at ranks 256 .. 256 + N - 1: no 2-byte token is a
                 prefix or suffix of it, so it can never be formed by a merge; every real merge's rank moves up by N
So every real id at or past the first shifted id moves up by N and nothing else changes:
    ids_derived(t) == [i if i < first else i + N for i in ids_committed(t)]
The committed upstream goldens, mapped, are then an exact reference for the derived model at ids past 65 535.

The derivation is pure Python (the GPU tests rebuild the models from the committed files at run time, so nothing large
is committed).  Run as a script, this file checks every derived model against upstream pip sentencepiece 0.2.1 /
tiktoken 0.12.0 over all committed goldens plus a bulk text set, and writes tests/golden/wide_goldens.json: a few
hundred texts with their ids frozen from upstream on the derived models, and the SHA-256 of each derived model's bytes
(so a test can prove it rebuilt exactly the model upstream was run on).
"""
import base64
import hashlib
import json
import os
import random
import struct
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

# name -> (committed model, filler count).  The three sp_bpe_8k boundary models have 65 534 pieces (the last one
# whose ids fit the 16-bit kernels; top id 65 533), 65 535 (the first one that takes the wide kernels; top id 65 534,
# still a uint16) and 65 536 (the first one whose ids do not all fit a uint16).
WIDE_FILL = 70000
DERIVED = {
    "sp_bpe_8k": ("sp_bpe_8k", WIDE_FILL),
    "sp_natural_32k": ("sp_natural_32k", WIDE_FILL),
    "sp_unigram_4k": ("sp_unigram_4k", WIDE_FILL),
    "sp_unigram_4k_bf": ("sp_unigram_4k_bf", WIDE_FILL),
    "tiktoken_1k": ("tiktoken_1k", WIDE_FILL),
    "sp_bpe_8k@65534": ("sp_bpe_8k", 65534 - 8000),
    "sp_bpe_8k@65535": ("sp_bpe_8k", 65535 - 8000),
    "sp_bpe_8k@65536": ("sp_bpe_8k", 65536 - 8000),
}


# ---------------------------------------------------------------------------- protobuf wire format
def _varint(buf, i):
    v = s = 0
    while True:
        b = buf[i]
        i += 1
        v |= (b & 0x7F) << s
        s += 7
        if b < 0x80:
            return v, i


def _put_varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _fields(buf):
    """(field number, wire type, value or payload, the whole record's bytes) of each field of one message."""
    i = 0
    while i < len(buf):
        start = i
        key, i = _varint(buf, i)
        num, wt = key >> 3, key & 7
        if wt == 0:
            val, i = _varint(buf, i)
        elif wt == 1:
            val, i = buf[i:i + 8], i + 8
        elif wt == 2:
            n, i = _varint(buf, i)
            val, i = buf[i:i + n], i + n
        elif wt == 5:
            val, i = buf[i:i + 4], i + 4
        else:
            raise ValueError("unsupported wire type %d" % wt)
        yield num, wt, val, buf[start:i]


def _piece(payload):
    """ModelProto.SentencePiece {1: piece, 2: score (float), 3: type (NORMAL = 1 by default)}"""
    s, score, typ = b"", 0.0, 1
    for num, wt, val, _ in _fields(payload):
        if num == 1 and wt == 2:
            s = bytes(val)
        elif num == 2 and wt == 5:
            score = struct.unpack("<f", val)[0]
        elif num == 3 and wt == 0:
            typ = val
    return s, score, typ


def _f32(x):
    return struct.unpack("<f", struct.pack("<f", x))[0]


def _interleaved_scores(real_scores, n):
    """n float32 scores spread evenly over the gaps between the distinct real scores, highest first."""
    d = sorted(set(real_scores), reverse=True)
    gaps = len(d) - 1
    out = []
    for g in range(gaps):
        c = (g + 1) * n // gaps - g * n // gaps
        for j in range(c):
            out.append(_f32(d[g] + (d[g + 1] - d[g]) * (j + 1) / (c + 1)))
    return out


def sp_filler(i):
    return (chr(0xF0000 + i // 300) + chr(0xF0000 + i % 300)).encode()


def derive_sp(blob, n_fill):
    """SentencePiece ModelProto bytes -> (derived bytes, first shifted id)."""
    recs = list(_fields(bytes(blob)))
    pieces = [_piece(val) for num, wt, val, _ in recs if num == 1 and wt == 2]
    first = next(i for i, p in enumerate(pieces) if p[2] == 1)
    scores = _interleaved_scores([p[1] for p in pieces if p[2] == 1], n_fill)
    fill = bytearray()
    for i, sc in enumerate(scores):
        s = sp_filler(i)
        body = b"\x0a" + _put_varint(len(s)) + s + b"\x15" + struct.pack("<f", sc)
        fill += b"\x0a" + _put_varint(len(body)) + body
    out, k = bytearray(), 0
    for num, wt, _, raw in recs:
        if num == 1 and wt == 2:
            if k == first:
                out += fill
            k += 1
        out += raw
    return bytes(out), first


def derive_tiktoken(text, n_fill):
    """tiktoken vocabulary file bytes (`base64 rank` lines) -> (derived bytes, first shifted id = 256)."""
    lines = [ln.split(b" ") for ln in bytes(text).split(b"\n") if ln.strip()]
    out = [ln for ln in lines if int(ln[1]) < 256]
    for i in range(n_fill):
        tok = bytes([0xF8 + (i >> 16), (i >> 8) & 0xFF, i & 0xFF])
        out.append([base64.b64encode(tok), str(256 + i).encode()])
    out += [[ln[0], str(int(ln[1]) + n_fill).encode()] for ln in lines if int(ln[1]) >= 256]
    return b"".join(a + b" " + r + b"\n" for a, r in out), 256


def derive(name, golden_dir=HERE):
    """name (a DERIVED key) -> (model file bytes, extra files {name: bytes}, first shifted id, filler count)."""
    base, n_fill = DERIVED[name]
    d = os.path.join(golden_dir, base)
    with open(os.path.join(d, "tokenizer.model"), "rb") as f:
        blob = f.read()
    extra = {}
    if os.path.exists(os.path.join(d, "tokenizer_config.json")):
        with open(os.path.join(d, "tokenizer_config.json"), "rb") as f:
            extra["tokenizer_config.json"] = f.read()
    model, first = (derive_tiktoken if base.startswith("tiktoken") else derive_sp)(blob, n_fill)
    return model, extra, first, n_fill


def write_derived(name, out_dir, golden_dir=HERE):
    """Writes the derived model directory; returns (first shifted id, filler count, model bytes)."""
    model, extra, first, n_fill = derive(name, golden_dir)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "tokenizer.model"), "wb") as f:
        f.write(model)
    for k, v in extra.items():
        with open(os.path.join(out_dir, k), "wb") as f:
            f.write(v)
    return first, n_fill, model


def map_ids(ids, first, n_fill):
    return [i if i < first else i + n_fill for i in ids]


def committed_goldens(base, golden_dir=HERE):
    """[(text bytes, ids)] of the committed upstream goldens of a committed model."""
    if base == "sp_bpe_8k":
        with open(os.path.join(golden_dir, "sp_bpe_8k_goldens.json")) as f:
            return [(bytes.fromhex(c["text"]), c["ids"]) for c in json.load(f)["cases"]]
    if base == "sp_natural_32k":
        with open(os.path.join(golden_dir, "natural_goldens.json")) as f:
            return [(bytes.fromhex(c["text"]), c["sp"]) for c in json.load(f)["cases"]]
    if base.startswith("sp_unigram"):
        with open(os.path.join(golden_dir, "sp_unigram_goldens.json")) as f:
            return [(bytes.fromhex(c["text"]), c["ids"]) for c in json.load(f)["cases"][base]]
    with open(os.path.join(golden_dir, "tiktoken_goldens.json")) as f:
        return [(bytes.fromhex(c["text"]), c["ids"]) for c in json.load(f)["cases"]]


# ---------------------------------------------------------------------------- texts
TIKTOKEN_NO_RANK = {0x00, 0x7F, 0xF5}   # bytes the tiktoken fixture leaves without a rank (upstream panics on them)


def golden_texts(name):
    """The texts frozen in wide_goldens.json for one derived model: short sentences, odd chars, memo-length words and,
    for the sp_bpe_8k family, texts that produce the model's top id (its last piece, 'v')."""
    sys.path.insert(0, ROOT)
    from xllm_service_b200 import workload
    rnd = random.Random(sum(map(ord, name)))
    texts = [s.encode() for s in workload.sentences(32, (1, 12), seed=41)]
    texts += [b"", b" ", b"a", "café naïve 日本語".encode(), "\U0001F642 x".encode(), b"don't 12345",
              b"  two  spaces ", b"aaaaaaaaaaaaaaa", b"bbbbbbbbbbbbbbbb", b"zqxjkvwpyfghmnb", "▁ ▁▁".encode(),
              b"\xff\xfe broken \xe6\x97"]
    for _ in range(12):
        texts.append(" ".join("".join(rnd.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(rnd.randint(1, 16)))
                              for _ in range(rnd.randint(1, 8))).encode())
    if name.startswith("sp_bpe_8k"):
        texts += [b"v", b"xv", b"v v v", b"xvx xv vx", b"av bv cv dv ev"]
    if name.startswith("tiktoken"):
        texts = [t for t in texts if not TIKTOKEN_NO_RANK & set(t)]
    return texts


def bulk_texts():
    """Check texts for the upstream comparison: workload sentences of every length plus random words."""
    sys.path.insert(0, ROOT)
    from xllm_service_b200 import workload
    rnd = random.Random(7)
    texts = [s.encode() for s in workload.sentences(1200, (1, 60), seed=19)]
    alphabet = list("abcdefghijklmnopqrstuvwxyz     ") + ["é", "日", "\t", "Q", "7", "▁", "\U0001F642", "\n"]
    texts += ["".join(rnd.choice(alphabet) for _ in range(rnd.randrange(0, 120))).encode() for _ in range(400)]
    return texts


# ---------------------------------------------------------------------------- generator
def _upstream(name, model):
    if DERIVED[name][0].startswith("tiktoken"):
        import tiktoken
        ranks = {}
        for ln in model.split(b"\n"):
            if ln.strip():
                a, r = ln.split(b" ")
                ranks[base64.b64decode(a)] = int(r)
        enc = tiktoken.Encoding(name, pat_str=r"[\s\S]+", mergeable_ranks=ranks, special_tokens={})
        return lambda t: enc._encode_single_piece(t) if t else [], len(ranks), len(set(ranks.values()))
    import sentencepiece as spm
    sp = spm.SentencePieceProcessor(model_proto=model)
    n_ranks = len({sp.GetScore(i) for i in range(sp.GetPieceSize()) if not (sp.IsUnknown(i) or sp.IsControl(i) or
                                                                            sp.IsByte(i))})
    return lambda t: sp.EncodeAsIds(t), sp.GetPieceSize(), n_ranks


def main():
    import sentencepiece as spm
    import tiktoken
    out = {"sentencepiece_version": spm.__version__, "tiktoken_version": tiktoken.__version__, "models": {}}
    bulk = bulk_texts()
    for name, (base, n_fill) in DERIVED.items():
        model, _, first, _ = derive(name)
        enc, n_pieces, n_ranks = _upstream(name, model)
        with open(os.path.join(HERE, base, "tokenizer.model"), "rb") as f:
            small = f.read()
        # 1. the committed goldens, mapped
        gold = committed_goldens(base)
        bad = [t[:40] for t, ids in gold if enc(t) != map_ids(ids, first, n_fill)]
        assert not bad, (name, len(bad), bad[:3])
        # 2. a bulk text set against upstream on the committed model, mapped
        if base.startswith("tiktoken"):
            import tiktoken as tk
            ranks = {}
            for ln in small.split(b"\n"):
                if ln.strip():
                    a, r = ln.split(b" ")
                    ranks[base64.b64decode(a)] = int(r)
            e0 = tk.Encoding(base, pat_str=r"[\s\S]+", mergeable_ranks=ranks, special_tokens={})
            enc0 = lambda t: e0._encode_single_piece(t) if t else []   # noqa: E731
            check = [t for t in bulk if not TIKTOKEN_NO_RANK & set(t)]
        else:
            s0 = spm.SentencePieceProcessor(model_proto=small)
            enc0 = s0.EncodeAsIds
            check = bulk
        bad = [t[:40] for t in check if enc(t) != map_ids(enc0(t), first, n_fill)]
        assert not bad, (name, len(bad), bad[:3])
        texts = golden_texts(name)
        cases = [{"text": t.hex(), "ids": enc(t)} for t in texts]
        top = n_pieces - 1
        if name.startswith("sp_bpe_8k"):
            assert any(top in c["ids"] for c in cases), name
        out["models"][name] = {"base": base, "n_fill": n_fill, "first_shifted": first, "n_pieces": n_pieces,
                               "n_ranks": n_ranks, "sha256": hashlib.sha256(model).hexdigest(), "cases": cases}
        print("%-18s pieces %6d  distinct ranks %6d  checked %4d goldens + %4d bulk texts  frozen %d" %
              (name, n_pieces, n_ranks, len(gold), len(check), len(cases)))
    with open(os.path.join(HERE, "wide_goldens.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
