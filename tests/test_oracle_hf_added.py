"""The HF oracle (oracle/hf_bpe_oracle.cc + oracle/oracle.py) on added-token sets of real sizes and shapes
(tests/golden/make_hf_added_fixture.py): the derived tokenizer.json files are byte-exact, the oracle reproduces the
goldens frozen from pip `tokenizers` 0.22.2 (two-pass split of normalized / non-normalized tokens, the ids the library
gives added tokens, decode through the ByteLevel decoder with lossy UTF-8), agrees with the wheel on a live fuzz when
it is importable, and the loader's limits (2048 tokens, 65 535 token bytes, 64 bytes per token) hold exactly."""
import json
import os
import random
import sys

import pytest

HERE = os.path.dirname(__file__)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_hf_added_fixture as fx  # noqa: E402

with open(fx.GOLD, encoding="utf-8") as f:
    GOLD = json.load(f)


@pytest.fixture(scope="module")
def derived(tmp_path_factory):
    d = tmp_path_factory.mktemp("hf_added")
    return {name: fx.write(name, str(d)) for name in fx.SETS}


def test_derived_files_are_byte_exact():
    assert sorted(GOLD["sets"]) == sorted(fx.SETS)
    for name in fx.SETS:
        assert fx.sha256(name) == GOLD["sets"][name]["sha256"], name
    assert len(fx.TOKENS["llama3_256"]()) == 256 and len(fx.TOKENS["wide_256"]()) == 256
    assert len(fx.TOKENS["deepseek_800"]()) >= 790
    assert 20_000 < sum(len(c.encode()) for c, _, _, _ in fx.TOKENS["deepseek_800"]()) < 30_000
    assert os.path.getsize(fx.GOLD) < 250_000


@pytest.mark.parametrize("name", fx.SETS)
def test_oracle_matches_goldens(oracle, derived, name):
    h = oracle.HfBpeOracle(derived[name])
    g = GOLD["sets"][name]
    assert h.vocab_size_with_added == g["vocab_size"]
    assert [h.token_to_id(c) for c, _, _, _ in fx.TOKENS[name]()] == g["token_ids"]
    bad = [s for s, ids in g["cases"] if h.prefix_ids + h.encode(s.encode()).tolist() + h.suffix_ids != ids]
    assert not bad, (len(bad), bad[:5])
    for ids, plain, skipped in g["decode"]:
        assert h.decode(ids) == plain and h.decode(ids, skip_special_tokens=True) == skipped, ids


def test_the_four_library_rules(oracle, derived):
    """Normalized tokens only between the others, ids as the library gives them, non-special tokens kept by
    decode(skip_special_tokens), added tokens through the ByteLevel decoder with lossy UTF-8."""
    h = oracle.HfBpeOracle(derived["gpt2_adv"])
    tid = h.token_to_id
    assert h.encode(b"yzab").tolist() == h.encode(b"y").tolist() + [tid("zab")]
    assert h.encode(b"kqwv").tolist() == [tid("kqw")] + h.encode(b"v").tolist()
    assert h.encode(b"<n>x").tolist() == [tid("<n>x")]                  # between them, leftmost-longest again
    assert h.encode(b"zoo").tolist() == h.encode(b"z").tolist() + [tid("oo")]
    assert h.encode(b"<b>").tolist() == h.encode(b"<").tolist() + [tid("b>")]
    assert tid("<qq>") != 9000 and tid("<zz>") != 5000 and tid("<qq>") >= 8000 and tid("<zz>") >= 8000
    assert tid("a") == h._vocab_id("a") and tid("é") == h._vocab_id("é")
    assert h.decode([tid("<tool>")], skip_special_tokens=True) == "<tool>"
    assert h.decode([tid("<a>")], skip_special_tokens=True) == ""
    assert h.decode([tid("Ġthe")]) == " the" and h.decode([tid("café")]) == "caf�"
    assert h.decode([tid("é")]) == "�" and h.decode([tid("<｜x｜>")]) == "<｜x｜>"


@pytest.mark.parametrize("name", fx.SETS)
def test_live_against_tokenizers_wheel(oracle, derived, name):
    tokenizers = pytest.importorskip("tokenizers")
    tok = tokenizers.Tokenizer.from_file(os.path.join(derived[name], "tokenizer.json"))
    h = oracle.HfBpeOracle(derived[name])
    assert tok.get_vocab_size(True) == h.vocab_size_with_added
    rnd = random.Random(fx.hash_seed(name) + 7)
    toks = [c for c, _, _, _ in fx.TOKENS[name]()]
    sample = toks if len(toks) <= 64 else rnd.sample(toks, 64)
    texts = fx.texts(name, rnd, 5000, sample)
    bad = [s for s in texts if h.prefix_ids + h.encode(s.encode()).tolist() + h.suffix_ids != tok.encode(s).ids]
    assert not bad, (len(bad), bad[:5])
    for s in texts[::50]:
        ids = tok.encode(s).ids
        assert h.decode(ids) == tok.decode(ids, skip_special_tokens=False), s
        assert h.decode(ids, skip_special_tokens=True) == tok.decode(ids, skip_special_tokens=True), s


def _limit_set(tmp_path, name, contents):
    with open(os.path.join(HERE, "golden", "hf_bpe_8k", "tokenizer.json"), encoding="utf-8") as f:
        d = json.load(f)
    d["added_tokens"] = [fx.entry(c, 8000 + i, True, False) for i, c in enumerate(contents)]
    p = tmp_path / name
    p.mkdir()
    (p / "tokenizer.json").write_text(json.dumps(d, ensure_ascii=False), encoding="utf-8")
    return str(p)


def limit_sets():
    """(name, contents, accepted): exactly at each limit of the loader, and one past it."""
    def sized(n, total):      # n distinct tokens of up to 64 bytes, `total` bytes in all
        out = ["<t%d|" % i for i in range(n)]
        left = total - sum(len(c) for c in out)
        for i in range(n):
            pad = min(64 - len(out[i]), left)
            out[i] += "x" * pad
            left -= pad
        assert left == 0
        return out
    return [("n2048_b65535", sized(2048, 65535), True), ("n2049", sized(2049, 40000), False),
            ("b65536", sized(2048, 65536), False), ("len64", ["<" + "y" * 62 + ">"], True),
            ("len65", ["<" + "y" * 63 + ">"], False), ("len64_utf8", ["<" + "日" * 20 + "y" + ">"], True)]


def test_limits_are_accepted_or_refused(tmp_path):
    import __graft_entry__ as ge
    ge.build()
    import xllm_service_b200 as x
    from xllm_service_b200 import _lib
    for name, contents, ok in limit_sets():
        assert len(set(contents)) == len(contents)
        path = _limit_set(tmp_path, name, contents)
        if ok:
            info = _lib.tokenizer_probe(path)
            assert info["split_mode"] == 3 and info["n_pieces"] == 8000 + len(contents), name
        else:
            with pytest.raises(x.IngestError) as e:
                _lib.tokenizer_probe(path)
            assert e.value.code == -5, name       # XLLM_ERR_UNSUPPORTED
    # a content listed twice: an identical repeat is the same token, one with other flags is refused
    with open(os.path.join(HERE, "golden", "hf_bpe_8k", "tokenizer.json"), encoding="utf-8") as f:
        d = json.load(f)
    for name, second, ok in (("repeat_same", fx.entry("<x>", 8000, True, False), True),
                             ("repeat_special", fx.entry("<x>", 8000, False, False), False),
                             ("repeat_normalized", fx.entry("<x>", 8000, True, True), False)):
        d["added_tokens"] = [fx.entry("<x>", 8000, True, False), second]
        p = tmp_path / name
        p.mkdir()
        (p / "tokenizer.json").write_text(json.dumps(d), encoding="utf-8")
        if ok:
            assert _lib.tokenizer_probe(str(p))["n_pieces"] == 8001
        else:
            with pytest.raises(x.IngestError) as e:
                _lib.tokenizer_probe(str(p))
            assert e.value.code == -5, name
    # under normalizer NFC a normalized token must be NFC-inert (the library matches NFC(content)); a non-normalized
    # one is matched on the raw text and may hold anything
    d["normalizer"] = {"type": "NFC"}
    for name, tok, ok in (("nfc_inert", fx.entry("<café>", 8000, False, True), True),
                          ("nfc_decomposed", fx.entry("<cafe\u0301>", 8000, False, True), False),
                          ("nfc_mark_raw", fx.entry("<cafe\u0301>", 8000, True, False), True)):
        d["added_tokens"] = [tok]
        p = tmp_path / name
        p.mkdir()
        (p / "tokenizer.json").write_text(json.dumps(d), encoding="utf-8")
        if ok:
            assert _lib.tokenizer_probe(str(p))["n_pieces"] == 8001, name
        else:
            with pytest.raises(x.IngestError) as e:
                _lib.tokenizer_probe(str(p))
            assert e.value.code == -5, name
    for name in fx.SETS:                          # every derived set loads, with the library's ids
        info = _lib.tokenizer_probe(fx.write(name, str(tmp_path / "sets")))
        assert info["n_pieces"] == max(GOLD["sets"][name]["token_ids"] + [GOLD["sets"][name]["vocab_size"] - 1]) + 1
