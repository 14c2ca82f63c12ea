#!/usr/bin/env python3
"""Micro-benchmark of the chained block-hash kernel alone (inputs resident in HBM).
Algorithmic bytes = 528 B per block (512 read + 16 written)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import xllm_service_b200 as x  # noqa: E402
from bench import peaks  # noqa: E402

PEAK_GBPS, PEAK_SRC = peaks()

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=65536)
ap.add_argument("--T", type=int, default=4096)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
a = ap.parse_args()

h = x.Ingest()
n, T = a.n, a.T
toks = torch.randint(0, 152000, (n, T), dtype=torch.int32, device="cuda")
tok_start = torch.arange(n, device="cuda", dtype=torch.int64) * T
n_tok = torch.full((n,), T, dtype=torch.int32, device="cuda")
nb = T // 128
key_start = torch.arange(n, device="cuda", dtype=torch.int64) * nb
keys = torch.zeros((n, nb, 16), dtype=torch.uint8, device="cuda")
stream = torch.cuda.Stream()  # a NULL stream argument would select the handle's own stream
torch.cuda.synchronize()
torch.cuda.set_stream(stream)
s = stream.cuda_stream
assert s != 0


def run():
    h.hash_blocks_device(n, toks.data_ptr(), tok_start.data_ptr(), n_tok.data_ptr(), keys.data_ptr(),
                         key_start.data_ptr(), s)


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
ms = sorted(ts)[len(ts) // 2]
byts = n * nb * 528
print(json.dumps({"kernel": "xxh3_chain128", "n": n, "T": T, "ms_median": ms, "ms_min": min(ts),
                  "GBps": byts / ms / 1e6, "frac_of_peak": byts / ms / 1e6 / PEAK_GBPS, "peak_source": PEAK_SRC,
                  "req_per_s": n / ms * 1e3}))
