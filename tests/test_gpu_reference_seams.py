"""The drop-in boundary exercised through the reference's OWN code (oracle/_ref/reference_seams_test, built by
oracle/build_ref.sh from tests/cpp/reference_seams_main.cc — it needs the reference checkout's headers, so the binary is
prebuilt in the build container and travels to the GPU box like the .so files):
  * the reference's tokenizer/fast_tokenizer.cpp, compiled UNMODIFIED and linked against libxllm_ingest.so, runs the
    pip-`tokenizers` goldens through FastTokenizer::encode / decode / token_to_id / id_to_token / vocab_size / clone;
  * host/reference_adaptors.h's GpuTokenizer — a subclass of the reference's real Tokenizer — does the same for a
    SentencePiece model, and hands requests the device refuses (non-NFC text under `normalizer: NFC`) to the wrapped
    stock tokenizer instead of failing them;
  * GpuCacheAwareRouting — a real LoadBalancePolicy subclass — picks the same prefill / decode instance names as the
    reference's own CacheAwareRouting over GlobalKVCacheMgr (libxllm_ref.so) on the same events and requests."""
import json
import os
import struct
import subprocess

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
ROOT = os.path.dirname(HERE)
EXE = os.path.join(ROOT, "oracle", "_ref", "reference_seams_test")


def _need_exe():
    if not os.path.exists(EXE):
        pytest.skip("oracle/_ref/reference_seams_test not built (bash oracle/build_ref.sh in the build container)")


def _run(args, texts, tmp_path):
    pf = tmp_path / "cases.bin"
    with open(pf, "wb") as f:
        for t in texts:
            f.write(struct.pack("<I", len(t)) + t)
    p = subprocess.run([EXE] + [a if a != "@cases" else str(pf) for a in args], capture_output=True, text=True,
                       timeout=600)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), (p.stdout[-1500:], p.stderr[-1500:])
    return p.stdout.strip().split("\n")


def _parse(lines):
    """-> vocab, [dict(ids, dec, tok)] in case order, trailer dict"""
    vocab = int(lines[0].split()[1])
    cases, trailer = [], {}
    for ln in lines[1:]:
        f = ln.split(" ")
        if f[0] == "ids":
            cases.append({"ids": [int(v) for v in f[2:2 + int(f[1])]] if f[1] != "FAIL" else None})
        elif f[0] == "dec":
            cases[-1]["dec"] = bytes.fromhex(f[1]) if len(f) > 1 else b""
        elif f[0] == "tok":
            cases[-1]["tok"] = (int(f[1]), bytes.fromhex(f[2]) if len(f) > 2 else b"")
        elif f[0] in ("unknown", "delegated"):
            trailer[f[0]] = int(f[1])
    return vocab, cases, trailer


@pytest.mark.parametrize("fixture", ["hf_bpe_8k", "hf_llama3_style", "hf_qwen2_style"])
def test_reference_fast_tokenizer_links_and_matches_goldens(fixture, tmp_path):
    _need_exe()
    if fixture == "hf_bpe_8k":
        g = json.load(open(os.path.join(HERE, "golden", "hf_bpe_goldens.json")))
        cases, vocab = g["cases"], g["vocab_size"]
    else:
        cases, vocab = json.load(open(os.path.join(HERE, "golden", "hf_cl100k_goldens.json")))["cases"][fixture], None
    texts = [bytes.fromhex(c["text"]) for c in cases]
    # FastTokenizer is constructed with the tokenizer.json path itself (tokenizer_factory.cpp:14-19)
    lines = _run(["fast", os.path.join(HERE, "golden", fixture, "tokenizer.json"), "@cases"], texts, tmp_path)
    got_vocab, got, trailer = _parse(lines)
    if vocab is not None:
        assert got_vocab == vocab
    assert trailer["unknown"] == 0
    assert len(got) == len(cases)
    n_dec = 0
    for t, c, o in zip(texts, cases, got):
        if o["ids"] is None:      # NFC refusal: only where the text really is not NFC-inert
            assert fixture == "hf_qwen2_style"
            continue
        assert o["ids"] == c["ids"], t[:60]
        if fixture == "hf_bpe_8k":
            assert o["dec"] == t   # byte-level BPE round trip (no template in this fixture)
            n_dec += 1
        else:
            assert o["dec"].endswith(t)   # template prefix text + the prompt
        if o["ids"]:
            assert o["tok"][0] == o["ids"][0]   # token_to_id(id_to_token(id)) == id
    assert fixture != "hf_bpe_8k" or n_dec > 300


def test_gpu_tokenizer_subclass_and_fallback(oracle, tmp_path):
    _need_exe()
    g = json.load(open(os.path.join(HERE, "golden", "sp_bpe_8k_goldens.json")))
    cases = [c for c in g["cases"] if "ids" in c]
    texts = [bytes.fromhex(c["text"]) for c in cases]
    lines = _run(["gpu", os.path.join(HERE, "golden", "sp_bpe_8k"), "@cases"], texts, tmp_path)
    vocab, got, trailer = _parse(lines)
    assert vocab == g["vocab_size"] and trailer["delegated"] == 0
    for t, c, o in zip(texts, cases, got):
        assert o["ids"] == c["ids"], t[:60]
    # Qwen2 layout (normalizer NFC): a decomposed "e + combining acute" is refused by the device path and must be
    # served by the wrapped stock tokenizer (both by the tokenizer and by its clone), never failed
    texts = ["plain ascii".encode(), "café au lait".encode(), "xÅ".encode()]
    lines = _run(["gpu", os.path.join(HERE, "golden", "hf_qwen2_style"), "@cases"], texts, tmp_path)
    _, got, trailer = _parse(lines)
    H = oracle.HfBpeOracle(os.path.join(HERE, "golden", "hf_qwen2_style"))
    assert got[0]["ids"] == H.prefix_ids + H.encode(texts[0]).tolist() + H.suffix_ids
    for k in (1, 2):
        assert got[k]["ids"] == [1000000 + b for b in texts[k]]    # the stand-in's recognisable ids
    assert trailer["delegated"] == 4       # 2 refused texts x (tokenizer + its clone)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_gpu_cache_aware_routing_policy_equals_reference_policy(seed, tmp_path):
    _need_exe()
    p = subprocess.run([EXE, "route", str(seed)], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), (p.stdout[-2000:], p.stderr[-2000:])
    line = [ln for ln in p.stdout.split("\n") if ln.startswith("route checked")][0].split()
    stats = dict(zip(line[1::2], (int(v) for v in line[2::2])))
    assert stats["checked"] == 600 and stats["routed"] > 300 and stats["mismatched"] == 0
    assert stats["recycled_id"] == 1 and stats["overflow_id"] == -1
