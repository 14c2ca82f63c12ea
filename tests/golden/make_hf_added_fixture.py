#!/usr/bin/env python3
"""Added-token sets of the sizes and shapes real models ship, derived from the committed HF fixtures:

  gpt2_adv      hf_bpe_8k          ~50 adversarial tokens: prefix chains, overlaps, whitespace / digit / apostrophe
                                   tokens, multi-byte and 64-byte tokens, vocabulary entries, normalized and
                                   non-normalized tokens that overlap, special and non-special ones, and two tokens
                                   listed at ids the `tokenizers` library does not give them
  llama3_256    hf_llama3_style    the 256 Llama-3 special tokens, the template's BOS switched to <|begin_of_text|>
  qwen2_chat    hf_qwen2_style     Qwen2 chat / FIM / tool tokens, special and not, normalized and not (NFC model)
  deepseek_800  hf_deepseek_style  ~800 DeepSeek-V3 tokens with fullwidth bars and U+2581 (~25 KB of token bytes)
  wide_256      hf_natural_128k    256 tokens at ids 128 471 and up (ids past 65 535: the wide kernels)

No derived tokenizer.json is committed: `derive(name)` rebuilds each one byte for byte from its base, and the tests
check the bytes against the SHA-256 frozen here.  `main()` freezes tests/golden/hf_added_goldens.json from upstream
`tokenizers` (pip 0.22.2): per set the vocabulary size with added tokens, token_to_id of every token, texts with
their ids from encode(add_special_tokens=True), and decode with and without skip_special_tokens for a subset.
"""
import hashlib
import json
import os
import random

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "hf_added_goldens.json")

BASE = {"gpt2_adv": "hf_bpe_8k", "llama3_256": "hf_llama3_style", "qwen2_chat": "hf_qwen2_style",
        "deepseek_800": "hf_deepseek_style", "wide_256": "hf_natural_128k"}
SETS = tuple(BASE)
EOT = "<|endoftext|>"
LONG64 = "<|" + "long_token_" * 5 + "x" * 5 + "|>"          # 64 bytes, the longest the loader takes
assert len(LONG64.encode()) == 64

# text pieces of test_gpu_hf.py's random strings
ALPHABET = list("abcdefghij  \t\n'.,!?012") + [
    "é", "日", "Σ", "١", " ", "　", "\U0001F600", "'s", "'re", " '", "<|endoftext|>", "\r\n", " ", "_",
    "²", "", " ", " ", " ", " ", "ǅ", "Ⅷ", "́", "﻿", "​", "­", "᠎",
    "⁠", "'ll", "'t", "'", "''", "!'", " 's", "\n's", "'S", "<|endoftext", "|>"]


def _gpt2_adv():
    """(content, special, normalized, listed id or None); None: the id the library gives it"""
    t = [(EOT, True, False, 0),
         ("<a>", True, False, None), ("<a>b", True, False, None), ("<a>bc", True, False, None),   # prefix chain
         ("foo", False, False, None), ("oob", False, False, None),                              # overlap
         ("ment", False, False, None),                                                         # inside words
         ("  ", False, False, None), ("\n\n", False, False, None), ("\t", False, False, None), (" x", False, False, None),
         ("'s", False, False, None), ("'", False, False, None), ("!'", False, False, None),
         ("123", False, False, None),
         ("é", False, False, None), ("日本", True, False, None), ("🙂", False, False, None), ("<｜x｜>", True, False, None),
         ("~", True, False, None),
         (LONG64, True, False, None),
         ("a", False, False, None),               # raw content is a vocabulary entry: the model's id
         ("Ġthe", False, False, None),            # spelled like a byte-level entry
         ("<tool>", False, False, None), ("café", False, False, None),
         # normalized tokens, matched only between the non-normalized ones
         ("zab", False, False, None), ("yza", False, True, None),           # "yzab": the non-normalized one wins
         ("kqw", False, False, None), ("qwv", False, True, None),           # "kqwv"
         ("oo", False, True, None), ("<n>", False, True, None), ("<n>x", True, True, None),
         ("<b", False, True, None), ("b>", False, False, None),            # "<b>"
         ("s!", False, True, None), ("  y", False, True, None), ("ll", True, True, None),
         ("<|eom|>", True, False, None), ("<|eom", False, True, None),
         ("\n", False, True, None), ("9", False, True, None),
         ("z" * 12 + "<|long", False, True, None),   # reaches into LONG64: the second pass must see all of that one
         ("<qq>", True, False, 9000),             # listed past the ids in use: the library gives 8000 + k
         ("<zz>", True, False, 5000)]             # listed at another entry's id
    return t


def _llama3():
    names = ["<|begin_of_text|>", "<|end_of_text|>", "<|reserved_special_token_0|>", "<|reserved_special_token_1|>",
             "<|finetune_right_pad_id|>", "<|reserved_special_token_2|>", "<|start_header_id|>", "<|end_header_id|>",
             "<|eom_id|>", "<|eot_id|>", "<|python_tag|>"]
    names += ["<|reserved_special_token_%d|>" % i for i in range(3, 3 + 256 - len(names))]
    return [(n, True, False, None) for n in names]


def _qwen2():
    sp = ["<|im_start|>", "<|im_end|>", "<|object_ref_start|>", "<|object_ref_end|>", "<|box_start|>", "<|box_end|>",
          "<|quad_start|>", "<|quad_end|>", "<|vision_start|>", "<|vision_end|>", "<|vision_pad|>", "<|image_pad|>",
          "<|video_pad|>"]
    ns = ["<tool_call>", "</tool_call>", "<|fim_prefix|>", "<|fim_middle|>", "<|fim_suffix|>", "<|fim_pad|>",
          "<|repo_name|>", "<|file_sep|>"]
    norm = ["<tool_response>", "</tool_response>", "<think>", "</think>", "<|im"]   # add_tokens(): normalized
    return ([(EOT, True, False, 0)] + [(s, True, False, None) for s in sp] + [(s, False, False, None) for s in ns] +
            [(s, False, True, None) for s in norm])


def _deepseek():
    b, u = "｜", "▁"
    t = [("<" + b + "begin" + u + "of" + u + "sentence" + b + ">", True, False, None),
         ("<" + b + "end" + u + "of" + u + "sentence" + b + ">", True, False, None),
         ("<" + b + u + "pad" + u + b + ">", True, False, None)]
    t += [("<" + b + "place" + u + "holder" + u + "no" + u + str(i) + b + ">", True, False, None) for i in range(784)]
    for w in ("fim" + u + "hole", "fim" + u + "begin", "fim" + u + "end", "tool" + u + "calls" + u + "begin",
              "tool" + u + "calls" + u + "end", "tool" + u + "call" + u + "begin", "tool" + u + "sep"):
        t.append(("<" + b + w + b + ">", True, False, None))
    for w in ("User", "Assistant", "tool" + u + "outputs" + u + "begin", "tool" + u + "output" + u + "end"):
        t.append(("<" + b + w + b + ">", False, True, None))
    t += [("<think>", False, True, None), ("</think>", False, True, None)]
    return t


def _wide():
    t = [("<|extra_%d|>" % i, i % 3 == 0, i % 5 == 4, None) for i in range(250)]
    t += [("<|wide|>", True, False, None), ("日本語の", False, False, None), (" \n", False, True, None),
          ("1234", False, False, None), ("<|wide", False, True, None), ("ﬁ", True, False, None)]
    return t


TOKENS = {"gpt2_adv": _gpt2_adv, "llama3_256": _llama3, "qwen2_chat": _qwen2, "deepseek_800": _deepseek,
          "wide_256": _wide}


def library_ids(vocab, contents):
    """The ids `tokenizers` gives added tokens when it loads a file (AddedVocabulary::add_tokens, in list order): a
    content that is a model.vocab entry or an earlier added token keeps that id; any other content gets
    len(model.vocab), or one past the largest added id once that is at least len(model.vocab)."""
    given, out = {}, []
    for c in contents:
        if c in given:
            i = given[c]
        elif c in vocab:
            i = vocab[c]
        else:
            top = max(given.values(), default=None)
            i = len(vocab) if top is None or top < len(vocab) else top + 1
        given.setdefault(c, i)
        out.append(i)
    return out


def entry(content, i, special, normalized):
    return {"id": i, "content": content, "single_word": False, "lstrip": False, "rstrip": False,
            "normalized": normalized, "special": special}


def derive(name, base_dir=HERE):
    """The derived tokenizer.json of set `name`, as bytes (deterministic)."""
    with open(os.path.join(base_dir, BASE[name], "tokenizer.json"), encoding="utf-8") as f:
        d = json.load(f)
    toks = TOKENS[name]()
    ids = library_ids(d["model"]["vocab"], [c for c, _, _, _ in toks])
    d["added_tokens"] = [entry(c, i if listed is None else listed, s, n)
                         for (c, s, n, listed), i in zip(toks, ids)]
    if name == "llama3_256":
        tp = d["post_processor"]["processors"][1]
        bos = toks[0][0]
        tp["single"][0]["SpecialToken"]["id"] = bos
        for it in tp["pair"]:
            if "SpecialToken" in it:
                it["SpecialToken"]["id"] = bos
        tp["special_tokens"] = {bos: {"id": bos, "ids": [ids[0]], "tokens": [bos]}}
    return json.dumps(d, ensure_ascii=False, separators=(",", ":")).encode("utf-8")


def write(name, out_dir, base_dir=HERE):
    """Writes <out_dir>/<name>/tokenizer.json; returns the directory."""
    path = os.path.join(out_dir, name)
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "tokenizer.json"), "wb") as f:
        f.write(derive(name, base_dir))
    return path


def sha256(name, base_dir=HERE):
    return hashlib.sha256(derive(name, base_dir)).hexdigest()


def token_contexts(tok, other):
    """Texts that put one token in the places where matching and pre-tokenizing go wrong."""
    chars = list(tok)
    prefixes = ["".join(chars[:k]) for k in range(1, len(chars))]
    return [tok, tok + tok + other, tok + " " + other + "  " + tok + "\n" + other,
            "ab" + tok + "cd 12" + tok + "34 !" + tok + "? 日本" + tok + "語 don" + tok + "'t " + tok + "'s",
            " ".join(prefixes) + " | " + tok[1:] + "|" + "".join(prefixes[-1:]) + "x"]


def texts(name, rnd, n_random=150, tokens=None):
    """Per token, its contexts; then random strings over ALPHABET extended with the tokens and their prefixes."""
    toks = [c for c, _, _, _ in TOKENS[name]()] if tokens is None else tokens
    out = []
    for i, t in enumerate(toks):
        out += token_contexts(t, toks[(i * 7 + 3) % len(toks)])
    alpha = ALPHABET + toks + [t[:len(t) // 2] for t in toks] + [t[1:] for t in toks]
    if name == "qwen2_chat":
        alpha = [a for a in alpha if a not in ("ǅ", "﻿")]   # keep the random texts in NFC-inert territory
    for _ in range(n_random):
        out.append("".join(rnd.choice(alpha) for _ in range(rnd.randrange(0, 40))))
    return out


def golden_texts(name):
    """The texts frozen in the goldens (kept small: the tests run every token's contexts against the oracle, which is
    checked against the library live): the contexts of every token of the small sets and of 12 tokens of the large
    ones, every sixteenth other token alone, and random strings."""
    toks = [c for c, _, _, _ in TOKENS[name]()]
    rnd = random.Random(hash_seed(name))
    if len(toks) <= 64:
        return texts(name, rnd, 50, toks)
    pick = toks[:6] + toks[-6:]
    return texts(name, rnd, 40, pick) + toks[6:-6:16]


def hash_seed(name):
    return int(hashlib.sha256(name.encode()).hexdigest()[:8], 16)


def main():
    import tempfile
    import tokenizers
    from tokenizers import Tokenizer
    gold = {"tokenizers_version": tokenizers.__version__, "sets": {}}
    with tempfile.TemporaryDirectory() as tmp:
        for name in SETS:
            tok = Tokenizer.from_file(os.path.join(write(name, tmp), "tokenizer.json"))
            toks = [c for c, _, _, _ in TOKENS[name]()]
            cases = []
            for s in golden_texts(name):
                cases.append([s, tok.encode(s, add_special_tokens=True).ids])
            rnd = random.Random(hash_seed(name) + 1)
            dec = []
            for s in [c[0] for c in cases if c[1]][:: max(1, len(cases) // 30)][:30]:
                ids = tok.encode(s, add_special_tokens=True).ids
                dec.append([ids, tok.decode(ids, skip_special_tokens=False), tok.decode(ids, skip_special_tokens=True)])
            for _ in range(10):   # ids in any order, byte tokens cut inside a UTF-8 char
                ids = [rnd.randrange(tok.get_vocab_size(True)) for _ in range(rnd.randrange(1, 12))]
                dec.append([ids, tok.decode(ids, skip_special_tokens=False), tok.decode(ids, skip_special_tokens=True)])
            gold["sets"][name] = {
                "sha256": sha256(name), "vocab_size": tok.get_vocab_size(True),
                "token_ids": [tok.token_to_id(t) for t in toks], "cases": cases, "decode": dec}
    with open(GOLD, "w", encoding="utf-8") as f:
        json.dump(gold, f, ensure_ascii=False, separators=(",", ":"))
    print({k: len(v["cases"]) for k, v in gold["sets"].items()}, os.path.getsize(GOLD))


if __name__ == "__main__":
    main()
