"""What the tokenizer's launch plan (sp_encode_plan) tells its callers: the kernels each ingest_batch chunk enqueues,
and the warps the profile reports, which must be those of the kernel that actually ran."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)


def _handle(model, env):
    import xllm_service_b200 as x
    os.environ.update(env)
    try:
        return x.Ingest(tokenizer_path=os.path.join(HERE, "golden", model))
    finally:
        for k in env:
            os.environ.pop(k, None)


# tokenizer kernels per chunk: express (SentencePiece BPE, memo on, not warm) + buffer path + long words (BPE only)
@pytest.mark.parametrize("model,env,tokenizer_launches", [
    ("sp_bpe_8k", {}, 3),
    ("sp_bpe_8k", {"XLLM_SP_MEMO_SLOTS": "0"}, 2),
    ("sp_bpe_8k", {"XLLM_SP_WARM": "1"}, 2),
    ("hf_bpe_8k", {}, 2),
    ("tiktoken_1k", {}, 2),
    ("sp_unigram_4k", {}, 1),
])
def test_launches_per_chunk(model, env, tokenizer_launches):
    from xllm_service_b200 import workload
    texts = [s.encode() for s in workload.sentences(1100, (1, 12), seed=4)]
    b = workload.pack_prompts(texts)
    h = _handle(model, env)
    try:
        out = h.ingest_batch(b.text, b.offsets, 128, want_match=False)
        chunks, launches = h.last_batch_stats()
        assert chunks > 1
        assert launches == (tokenizer_launches + 2) * chunks   # + row prep + hash per chunk
        assert (out["status"] == 0).all()
        ids, n_ids, _ = h.encode_batch(b.text, b.offsets, 128)
        assert (out["n_ids"] == n_ids).all()
        assert all((out["ids"][r, :n_ids[r]] == ids[r, :n_ids[r]]).all() for r in range(b.n))
    finally:
        h.close()


def _oracle_encoder(oracle, model):
    d = os.path.join(HERE, "golden", model)
    if model.startswith("hf"):
        H = oracle.HfBpeOracle(d)
        return lambda t: H.prefix_ids + H.encode(t).tolist() + H.suffix_ids
    T = oracle.TiktokenOracle(d)
    return lambda t: T.encode(t).tolist()


@pytest.mark.parametrize("model", ["hf_bpe_8k", "tiktoken_1k"])
def test_profile_reports_the_warm_grid(oracle, model):
    """The warm-up kernel keeps 16-row lane columns, so more of its warps fit an SM than of the default kernel's
    32-row ones: the profile must size its per-warp buffer for, and report, the grid that ran."""
    from xllm_service_b200 import workload
    texts = [s.encode() for s in workload.sentences(16384, (1, 12), seed=9)]
    b = workload.pack_prompts(texts)
    stride = 128
    enc = _oracle_encoder(oracle, model)
    warps = {}
    for name, env in (("default", {}), ("warm", {"XLLM_SP_WARM": "1"})):
        h = _handle(model, env)
        try:
            n_ids, status, warp_ns = h.encode_batch_profile(b.text, b.offsets, stride)
            ids, n_ids2, status2 = h.encode_batch(b.text, b.offsets, stride)
        finally:
            h.close()
        assert (status == 0).all()
        assert (n_ids == n_ids2).all() and (status == status2).all()
        for r in range(0, b.n, 97):
            assert ids[r, :n_ids[r]].tolist() == enc(b.prompt(r)), (name, r)
        warps[name] = warp_ns.size
    assert warps["warm"] > warps["default"] > 0, warps
