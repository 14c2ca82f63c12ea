"""The per-launch word memo of the encode kernels (csrc/sp_encode.cu "word memo") must never change a result:
the same batches are encoded with the memo at its default size, squeezed into 4 slots (nearly every insert fails),
switched off, and through the wide (32-bit pair state, 28-bit memo ids) kernel variants — all equal to the CPU
oracle (sentencepiece_tokenizer.cpp:115-168 / fast_tokenizer.cpp:20-30 / tiktoken_tokenizer.cpp:115-294)."""
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
SP_DIR = os.path.join(HERE, "golden", "sp_bpe_8k")
HF_DIR = os.path.join(HERE, "golden", "hf_bpe_8k")
TK_DIR = os.path.join(HERE, "golden", "tiktoken_1k")

VARIANTS = [
    ("default", {}),
    ("tiny", {"XLLM_SP_MEMO_SLOTS": "4"}),
    ("off", {"XLLM_SP_MEMO_SLOTS": "0"}),
    ("wide", {"XLLM_SP_FORCE_WIDE": "1"}),
    ("wide_off", {"XLLM_SP_FORCE_WIDE": "1", "XLLM_SP_MEMO_SLOTS": "0"}),
    # the warm-up kernels (drain_pass with WARM: memo misses merged ahead in full rounds, long words resolved ahead into the
    # per-warp scratch), narrow and wide, and with a memo so small that the warm-up's inserts mostly fail
    ("warm", {"XLLM_SP_WARM": "1"}),
    ("warm_wide", {"XLLM_SP_WARM": "1", "XLLM_SP_FORCE_WIDE": "1"}),
    ("warm_tiny", {"XLLM_SP_WARM": "1", "XLLM_SP_MEMO_SLOTS": "4"}),
]


def _handle(model_dir, env):
    import xllm_service_b200 as x
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return x.Ingest(tokenizer_path=model_dir)   # the knobs are read when the handle is created
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def _encode_all(tok, texts):
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    stride = max(16, 3 * max((len(t) for t in texts), default=0) + 8)
    ids, n_ids, status = tok.encode_batch(b.text, b.offsets, stride)
    return [ids[i, :n_ids[i]].tolist() for i in range(len(texts))], status


def _texts(seed):
    """Heavy word repetition across and inside prompts (the memo's hit path), keys at the 15-byte limit,
    words with more ids than a memo entry holds, unknown chars, bare U+2581 words, duplicated spaces."""
    from xllm_service_b200 import workload
    rnd = random.Random(seed)
    vocab = [w.decode() for w in workload.make_vocabulary()[:300]]
    odd = ["a" * 14, "b" * 15, "c" * 16, "d" * 17, "zqxjkvwpyfgh", "zqxjkvwpyfghmn", "日本", "é", "naïve", "x1y2z3",
           "▁", "▁▁", "don't", "<|endoftext|>", "\x00", "ÿ", "🙂", "12345678901234", "Zq" * 7, "zq" * 8]
    out = []
    for i in range(160):
        words = []
        for _ in range(rnd.randrange(1, 400)):
            words.append(rnd.choice(odd) if rnd.random() < 0.15 else rnd.choice(vocab))
            if rnd.random() < 0.05:
                words.append("")          # a doubled space
        out.append(" ".join(words).encode())
    out += [b"", b" ", b"same same same same same same same same", ("word " * 3000).encode()]
    return out


@pytest.mark.parametrize("name,env", VARIANTS)
def test_sentencepiece_variants(oracle, name, env):
    sp = oracle.SentencePieceOracle(SP_DIR)
    texts = _texts(3)
    h = _handle(SP_DIR, env)
    try:
        for _ in range(2):                      # second launch: the memo starts empty again
            got, status = _encode_all(h, texts)
            assert (status == 0).all()
            bad = [t[:40] for t, g in zip(texts, got) if g != sp.encode(t).tolist()]
            assert not bad, (name, len(bad), bad[:3])
    finally:
        h.close()


@pytest.mark.parametrize("name,env", VARIANTS)
def test_hf_variants(oracle, name, env):
    hf = oracle.HfBpeOracle(HF_DIR)
    texts = _texts(4)
    h = _handle(HF_DIR, env)
    try:
        got, status = _encode_all(h, texts)
        assert (status == 0).all()
        bad = [t[:40] for t, g in zip(texts, got) if g != hf.encode(t).tolist()]
        assert not bad, (name, len(bad), bad[:3])
    finally:
        h.close()


@pytest.mark.parametrize("name,env", [VARIANTS[0], VARIANTS[3], VARIANTS[5]])
def test_tiktoken_variants(oracle, name, env):
    tk = oracle.TiktokenOracle(TK_DIR)
    texts = [t for t in _texts(5)[:40]]
    h = _handle(TK_DIR, env)
    try:
        got, status = _encode_all(h, texts)
        assert (status == 0).all()
        for t, g in zip(texts, got):
            assert g == tk.encode(t).tolist(), (name, t[:40])
    finally:
        h.close()


def test_pipeline_chunks_each_have_their_own_memo(oracle):
    """xllm_ingest_batch runs chunks concurrently on several streams; every chunk clears and fills its own table."""
    import xllm_service_b200 as x
    sp = oracle.SentencePieceOracle(SP_DIR)
    from xllm_service_b200 import workload
    texts = _texts(6) * 3
    b = workload.pack_prompts(texts)
    h = x.Ingest(tokenizer_path=SP_DIR)
    try:
        h.set_pipeline(17, 1 << 16)
        stride = 3 * max(len(t) for t in texts) + 8
        res = h.ingest_batch(b.text, b.offsets, stride, want_keys=False, want_match=False)
        ids, n_ids, status = res["ids"], res["n_ids"], res["status"]
        assert (status == 0).all()
        for i, t in enumerate(texts):
            assert ids[i, :n_ids[i]].tolist() == sp.encode(t).tolist(), i
    finally:
        h.close()


@pytest.mark.parametrize("model,kind", [(SP_DIR, "sp"), (HF_DIR, "hf")])
def test_memo_kept_across_launches(oracle, model, kind):
    """xllm_set_memo_policy(N): the table survives between launches (the service setting) and is cleared after N requests;
    different batches one after the other, through the single-launch entry point and through the chunk pipeline, all
    equal the oracle — a stale table is only ever less complete, never wrong."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    orc = oracle.SentencePieceOracle(model) if kind == "sp" else oracle.HfBpeOracle(model)
    h = x.Ingest(tokenizer_path=model)
    try:
        h.set_memo_policy(500)                  # three batches of 164 prompts stay on one table, the fourth clears it
        for seed in (11, 12, 11, 13, 14, 12):
            texts = _texts(seed)
            got, status = _encode_all(h, texts)
            assert (status == 0).all()
            bad = [t[:40] for t, g in zip(texts, got) if g != orc.encode(t).tolist()]
            assert not bad, (seed, len(bad), bad[:3])
        h.set_pipeline(23, 1 << 16)
        for seed in (21, 22, 21):
            texts = _texts(seed)
            b = workload.pack_prompts(texts)
            stride = 3 * max(len(t) for t in texts) + 8
            res = h.ingest_batch(b.text, b.offsets, stride, want_keys=False, want_match=False)
            assert (res["status"] == 0).all()
            for i, t in enumerate(texts):
                assert res["ids"][i, :res["n_ids"][i]].tolist() == orc.encode(t).tolist(), (seed, i)
        h.set_memo_policy(0)                    # back to a fresh table per launch
        got, status = _encode_all(h, _texts(31))
        assert (status == 0).all() and got == [orc.encode(t).tolist() for t in _texts(31)]
    finally:
        h.close()
