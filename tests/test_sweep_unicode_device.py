"""Exhaustive device-vs-oracle sweeps over every Unicode code point: all 1.1 M scalar values, each in five contexts
("a<c>b <c>1\n<c>"), through the CUDA normaliser / pre-tokenizers / merge kernels against the CPU oracle — 5 models,
part of `-m gpu` (also selectable alone with `-m sweep`).  The oracles themselves are swept against
the upstream wheels on CPU (tests/test_oracle_sp.py, tests/test_oracle_hf.py), so this is what separates the device
tables from the oracle's although both are generated from one Unicode data file."""
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.sweep, pytest.mark.gpu]
STRIDE = 256   # U+FDFA alone normalises to 18 chars; five copies with byte fallback need > 64 ids
HERE = os.path.dirname(__file__)


def _cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _texts():
    out = []
    for cp in range(1, 0x110000):
        if 0xD800 <= cp < 0xE000:
            continue
        ch = chr(cp)
        out.append(("a" + ch + "b " + ch + "1\n" + ch).encode())
    return out


def _run(model_dir, oracle_encode, accept_status=(0,)):
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    texts = _texts()
    b = workload.pack_prompts(texts)
    h = x.Ingest(tokenizer_path=model_dir)
    try:
        ids, n_ids, status = h.encode_batch(b.text, b.offsets, STRIDE)
    finally:
        h.close()
    bad = []
    for i, t in enumerate(texts):
        if status[i] not in accept_status:
            bad.append((i, int(status[i])))
            continue
        if status[i] == 0 and ids[i, :n_ids[i]].tolist() != oracle_encode(t):
            bad.append((i, t))
    assert not bad, (len(bad), bad[:10])


@pytest.mark.skipif(not _cuda(), reason="needs a CUDA device")
@pytest.mark.parametrize("name", ["sp_bpe_8k", "sp_unigram_4k_bf"])
def test_sentencepiece_every_code_point(oracle, name):
    d = os.path.join(HERE, "golden", name)
    S = oracle.SentencePieceOracle(d)
    _run(d, lambda t: S.encode(t).tolist())


@pytest.mark.skipif(not _cuda(), reason="needs a CUDA device")
@pytest.mark.parametrize("name", ["hf_bpe_8k", "hf_llama3_style", "hf_qwen2_style", "hf_deepseek_style"])
def test_hf_every_code_point(oracle, name):
    import unicodedata
    d = os.path.join(HERE, "golden", name)
    H = oracle.HfBpeOracle(d)

    def enc(t):
        if H.nfc and unicodedata.normalize("NFC", t.decode()) != t.decode():
            return None                      # must have been refused (-5), never tokenised
        return H.prefix_ids + H.encode(t).tolist() + H.suffix_ids
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    texts = _texts()
    b = workload.pack_prompts(texts)
    h = x.Ingest(tokenizer_path=d)
    try:
        ids, n_ids, status = h.encode_batch(b.text, b.offsets, STRIDE)
    finally:
        h.close()
    bad = []
    for i, t in enumerate(texts):
        want = enc(t)
        if want is None:
            if status[i] != -5:
                bad.append((i, "non-NFC accepted", int(status[i])))
        elif status[i] == -5 and H.nfc:
            pass                             # conservative refusal of an NFC text with a non-inert char: allowed
        elif status[i] != 0 or ids[i, :n_ids[i]].tolist() != want:
            bad.append((i, t, int(status[i])))
    assert not bad, (len(bad), bad[:10])
