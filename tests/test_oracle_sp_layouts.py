"""The CPU oracle (oracle/sp_oracle.cc) on the SentencePiece layouts of tests/golden/make_sp_layouts_fixture.py — kept
whitespace with U+2581-run pieces and the identity normaliser (Llama-2 / Mistral), no dummy prefix, cross-word BPE
pieces, long Unigram chains — against the goldens minted with pip sentencepiece 0.2.1, and live against the wheel when
it imports.  The loader must report the layout each fixture was built for."""
import hashlib
import importlib.util
import json
import os
import random

import pytest

HERE = os.path.dirname(__file__)
GOLD = os.path.join(HERE, "golden", "sp_layouts_goldens.json")


def _load_generator():
    spec = importlib.util.spec_from_file_location("make_sp_layouts_fixture",
                                                  os.path.join(HERE, "golden", "make_sp_layouts_fixture.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


ML = _load_generator()


@pytest.fixture(scope="module")
def gold():
    with open(GOLD) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def dirs(tmp_path_factory):
    root = tmp_path_factory.mktemp("sp_layouts")
    return {n: ML.materialise(n, root) for n in ML.NAMES}


@pytest.mark.parametrize("name", ML.NAMES)
def test_models_are_the_ones_upstream_ran(dirs, gold, name):
    """The committed models, and chain_unigram rebuilt from sp_unigram_4k, are byte for byte the models the goldens
    were minted on."""
    with open(os.path.join(dirs[name], "tokenizer.model"), "rb") as f:
        assert hashlib.sha256(f.read()).hexdigest() == gold["models"][name]["sha256"]


@pytest.mark.parametrize("name", ML.NAMES)
def test_oracle_equals_goldens(oracle, dirs, gold, name):
    S = oracle.SentencePieceOracle(dirs[name])
    cases = gold["models"][name]["cases"]
    assert len(cases) >= 60
    bad = [c["text"][:60] for c in cases if S.encode(bytes.fromhex(c["text"])).tolist() != c["ids"]]
    assert not bad, (len(bad), bad[:4])


@pytest.mark.parametrize("name", ML.NAMES)
def test_probe_reports_layout(dirs, gold, name):
    from xllm_service_b200 import _lib
    info = _lib.tokenizer_probe(dirs[name])
    for k, v in ML.LAYOUT[name].items():
        assert info[k] == v, (k, info[k], v)
    assert info["n_pieces"] == gold["models"][name]["n_pieces"]
    assert gold["models"][name]["split_mode"] == info["split_mode"]


def test_texts_reach_the_seams(gold):
    """The texts hold what the layouts are about: byte pieces for LF / tab / NUL under the identity normaliser, runs
    of 171+ spaces (Unigram words past 511 bytes), chains of 33+ a's in the goldens; prompts of 5-20 KB for the
    cross-word model and space runs past the 1 KB long-word threshold in the seam texts."""
    g = gold["models"]
    llama = [bytes.fromhex(c["text"]) for c in g["llama_bpe"]["cases"]]
    assert any(b"\n" in t for t in llama) and any(b"\x00" in t for t in llama) and any(b" " * 600 in t for t in llama)
    assert any(bytes.fromhex(c["text"]) == b"a" * 65 for c in g["chain_unigram"]["cases"])
    assert max(len(t) for t in ML.seam_texts("nosplit_bpe")) >= 20000
    assert any(b" " * 1100 in t for t in ML.seam_texts("llama_bpe"))
    assert gold["sentencepiece_version"] == "0.2.1"


def test_generator_layout_check_accepts_the_models(dirs):
    """The generator's own layout assertions (proto and loader) hold for the models."""
    pytest.importorskip("sentencepiece")
    for name in ML.NAMES:
        with open(os.path.join(dirs[name], "tokenizer.model"), "rb") as f:
            ML.check_layout(name, f.read(), dirs[name])


@pytest.mark.parametrize("name", ML.NAMES)
def test_live_against_sentencepiece_wheel(oracle, dirs, name):
    """The fuzz set, and the long seam texts the device tests check against the oracle."""
    spm = pytest.importorskip("sentencepiece")
    d = dirs[name]
    ref = spm.SentencePieceProcessor(model_file=os.path.join(d, "tokenizer.model"))
    S = oracle.SentencePieceOracle(d)
    rnd = random.Random(len(name))
    alphabet = list("abcdefghijklmnopqrstuvwxyz      \t\n\r0123456789") + [
        "\x00", "▁", "é", "日", "\U0001F600", "    ", "        ", "a" * 33, "b" * 40, "\r\n", "ﬁ", " "]
    for i in range(800):
        k = rnd.randrange(0, 120)
        t = bytes(rnd.getrandbits(8) for _ in range(k)) if i % 5 == 0 else \
            "".join(rnd.choice(alphabet) for _ in range(k)).encode()
        assert S.encode(t).tolist() == ref.EncodeAsIds(t), t
    for t in ML.seam_texts(name):
        assert S.encode(t).tolist() == ref.EncodeAsIds(t), t[:60]
