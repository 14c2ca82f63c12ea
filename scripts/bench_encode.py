#!/usr/bin/env python3
"""Micro-benchmark of the encode kernel alone (text resident in HBM).  --backend sp (default) times the
SentencePiece fixture on the exact-T workload; --backend hf times the HF byte-level BPE fixture on the same text
(token counts then differ per prompt) and, with --cpu, pip `tokenizers` (the Rust crate the reference links) on
the host cores for the same prompts."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import xllm_service_b200 as x  # noqa: E402
from bench import peaks  # noqa: E402

PEAK_GBPS, PEAK_SRC = peaks()
from xllm_service_b200 import workload  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=8192)
ap.add_argument("--T", type=int, default=4096)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--check", type=int, default=4)
ap.add_argument("--backend", choices=["sp", "hf", "unigram"], default="sp")
ap.add_argument("--hf-dir", default="hf_bpe_8k", help="fixture under tests/golden: hf_bpe_8k | hf_llama3_style | hf_qwen2_style")
ap.add_argument("--cpu", type=int, default=0, help="hf: prompts to time through pip tokenizers encode_batch")
a = ap.parse_args()

model = os.path.join(ROOT, "tests", "golden", "sp_bpe_8k")
h = x.Ingest(tokenizer_path=model)
hf_dir = os.path.join(ROOT, "tests", "golden", a.hf_dir)
uni_dir = os.path.join(ROOT, "tests", "golden", "sp_unigram_4k_bf")
h_run = x.Ingest(tokenizer_path=hf_dir) if a.backend == "hf" else (x.Ingest(tokenizer_path=uni_dir) if a.backend == "unigram" else h)
vocab = workload.make_vocabulary()
t0 = time.time()
wb = workload.pack_prompts(vocab)
_, wcnt, st = h.encode_batch(wb.text, wb.offsets, 32)
assert (st == 0).all()
batch, _ = workload.make_prompts_exact_tokens(a.n, a.T, wcnt, seed=1)
print("gen %.1fs, text bytes/prompt %.0f" % (time.time() - t0, batch.text.size / a.n), file=sys.stderr)

stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
d_text = torch.from_numpy(batch.text).cuda()
d_off = torch.from_numpy(batch.offsets).cuda()
stride = a.T + 64 if a.backend == "sp" else 2 * a.T
d_ids = torch.zeros((a.n, stride), dtype=torch.int32, device="cuda")
d_n = torch.zeros(a.n, dtype=torch.int32, device="cuda")
d_st = torch.zeros(a.n, dtype=torch.int32, device="cuda")
torch.cuda.synchronize()


def run():
    h_run.encode_batch_device(a.n, d_text.data_ptr(), d_off.data_ptr(), d_ids.data_ptr(), stride, d_n.data_ptr(),
                          d_st.data_ptr(), stream.cuda_stream)


for _ in range(a.warmup):
    run()
torch.cuda.synchronize()
ts = []
for _ in range(a.iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run()
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
assert (d_st.cpu().numpy() == 0).all(), d_st.cpu().numpy()[:10]
n_tok = int(d_n.sum().item())
if a.backend == "sp":
    assert (d_n.cpu().numpy() == a.T).all(), d_n.cpu().numpy()[:10]
extra = {}
if a.backend == "unigram":
    from oracle import oracle as o
    U = o.SentencePieceOracle(uni_dir)
    ids = d_ids[:a.check].cpu().numpy()
    cnt = d_n[:a.check].cpu().numpy()
    for i in range(a.check):
        assert ids[i, :cnt[i]].tolist() == U.encode(batch.prompt(i)).tolist()
elif a.backend == "hf":
    from oracle import oracle as o
    H = o.HfBpeOracle(hf_dir)
    ids = d_ids[:a.check].cpu().numpy()
    cnt = d_n[:a.check].cpu().numpy()
    for i in range(a.check):
        assert ids[i, :cnt[i]].tolist() == H.prefix_ids + H.encode(batch.prompt(i)).tolist() + H.suffix_ids
    if a.cpu:
        from tokenizers import Tokenizer
        ref = Tokenizer.from_file(os.path.join(hf_dir, "tokenizer.json"))
        texts = [batch.prompt(i).decode() for i in range(a.cpu)]
        ref.encode_batch(texts[:8])
        t0 = time.time()
        enc = ref.encode_batch(texts)
        dt = time.time() - t0
        got = d_ids[:a.cpu].cpu().numpy()
        gn = d_n[:a.cpu].cpu().numpy()
        for i in range(0, a.cpu, max(1, a.cpu // 64)):
            assert got[i, :gn[i]].tolist() == enc[i].ids
        extra = {"pip_tokenizers_req_per_s": a.cpu / dt, "pip_tokenizers_prompts": a.cpu, "host_cores": os.cpu_count()}
elif a.check:
    from oracle import oracle as o
    S = o.SentencePieceOracle(model)
    ids = d_ids[:a.check].cpu().numpy()
    for i in range(a.check):
        assert ids[i, :a.T].tolist() == S.encode(batch.prompt(i)).tolist()
ms = sorted(ts)[len(ts) // 2]
byts = batch.text.size + 4 * n_tok
print(json.dumps({"kernel": "sp_encode", "backend": a.backend, "tokens_per_prompt": n_tok / a.n, **extra, "n": a.n, "T": a.T, "ms_median": ms, "ms_min": min(ts),
                  "algo_GBps": byts / ms / 1e6, "frac_of_peak": byts / ms / 1e6 / PEAK_GBPS, "peak_source": PEAK_SRC,
                  "req_per_s": a.n / ms * 1e3, "text_bytes_per_prompt": batch.text.size / a.n}))
