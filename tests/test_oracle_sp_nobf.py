"""The CPU oracle (oracle/sp_oracle.cc) on the SentencePiece BPE models without byte fallback of
tests/golden/make_sp_nobf_fixture.py, against the goldens minted with pip sentencepiece 0.2.1, and live against the
wheel when it imports.  A char no piece covers is <unk>, and a run of unknown symbols is ONE <unk>: the merging of
consecutive unknown pieces (emit_piece), which the other BPE fixtures (all byte fallback) never reach."""
import hashlib
import importlib.util
import json
import os
import random

import pytest

HERE = os.path.dirname(__file__)
GOLD = os.path.join(HERE, "golden", "sp_nobf_goldens.json")


def _load_generator():
    spec = importlib.util.spec_from_file_location("make_sp_nobf_fixture",
                                                  os.path.join(HERE, "golden", "make_sp_nobf_fixture.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


MN = _load_generator()


@pytest.fixture(scope="module")
def gold():
    with open(GOLD, encoding="utf-8") as f:
        return json.load(f)


@pytest.fixture(scope="module")
def dirs(tmp_path_factory):
    root = tmp_path_factory.mktemp("sp_nobf")
    return {n: MN.materialise(n, root) for n in MN.NAMES}


@pytest.mark.parametrize("name", MN.NAMES)
def test_models_are_the_ones_upstream_ran(dirs, gold, name):
    """The committed models, and the nmt_nfkc ones with sp_bpe_8k's charsmap put back, are byte for byte the models
    the goldens were minted on."""
    with open(os.path.join(dirs[name], "tokenizer.model"), "rb") as f:
        assert hashlib.sha256(f.read()).hexdigest() == gold["models"][name]["sha256"]


def test_texts_are_the_generators(gold):
    assert [t.encode() for t in gold["texts"]] == MN.golden_texts()
    assert gold["sentencepiece_version"] == "0.2.1"


@pytest.mark.parametrize("name", MN.NAMES)
def test_oracle_equals_goldens(oracle, dirs, gold, name):
    S = oracle.SentencePieceOracle(dirs[name])
    g = gold["models"][name]
    bad = [t[:60] for t, ids in zip(gold["texts"], g["ids"]) if S.encode(t.encode()).tolist() != ids]
    assert not bad, (len(bad), bad[:4])


@pytest.mark.parametrize("name", MN.NAMES)
def test_goldens_hold_unknown_runs(gold, name):
    """The goldens reach the unknown-symbol seams: one <unk> for a run of 1..70 unknowns (never two in a row), runs
    inside words of 15..17 bytes, of 33..512 bytes and of more than 512 bytes; the seam texts, words past 2048."""
    g = gold["models"][name]
    unk = g["unk_id"]
    texts = gold["texts"]
    assert sum(ids.count(unk) for ids in g["ids"]) >= 700
    assert not any(a == b == unk for ids in g["ids"] for a, b in zip(ids, ids[1:]))
    runs = {len(t) - 4: ids for t, ids in zip(texts, g["ids"])
            if t.startswith("a ") and t.endswith(" b") and t[2:-2] and set(t[2:-2]) <= set(MN.UNKNOWN_ASCII)}
    assert sorted(runs) == list(range(1, 41))
    assert all(ids.count(unk) == 1 for ids in runs.values())
    longest = {len(w) for t in texts for w in t.split(" ") if any(c in w for c in MN.UNKNOWN_ASCII)}
    assert {15, 16, 17}.issubset(longest) and any(33 <= n <= 512 for n in longest) and max(longest) > 512
    assert max(len(w) for t in MN.seam_texts() for w in t.split(b" ")) > 2048


def test_generator_checks_accept_the_models(dirs):
    """The generator's own assertions on layout and unknown chars hold for the models."""
    pytest.importorskip("sentencepiece")
    for name in MN.NAMES:
        with open(os.path.join(dirs[name], "tokenizer.model"), "rb") as f:
            MN.check_model(name, f.read(), dirs[name])


@pytest.mark.parametrize("name", MN.NAMES)
def test_live_against_sentencepiece_wheel(oracle, dirs, name):
    """The long seam texts the device tests check against the oracle, a fuzz set rich in unknowns, runs of unknowns
    inside long words, and invalid UTF-8 (each bad byte is an unknown char), against the wheel."""
    spm = pytest.importorskip("sentencepiece")
    d = dirs[name]
    ref = spm.SentencePieceProcessor(model_file=os.path.join(d, "tokenizer.model"))
    S = oracle.SentencePieceOracle(d)
    rnd = random.Random(len(name))
    texts = MN.seam_texts() + MN.random_texts(rnd, 600, 120)
    texts += [bytes(rnd.getrandbits(8) for _ in range(rnd.randrange(1, 60))) for _ in range(100)]
    for n in (31, 32, 33, 100, 512, 513, 900, 2049):
        texts.append(("x " + MN.word_with_unknowns(rnd, n) + " y").encode())
    for t in texts:
        assert S.encode(t).tolist() == ref.EncodeAsIds(t), t[:60]
