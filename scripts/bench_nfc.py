#!/usr/bin/env python3
"""What exact NFC verification costs (csrc/hf_nfc.cu, xllm_set_nfc_policy(h, XLLM_NFC_VERIFY)) on the Qwen2-style
tokenizer.json (`normalizer: NFC`): 16 K prompts of 16 KB, device-resident, CUDA events around the whole encode call.

  multilingual  NFC text with combining marks in a dozen scripts (tests/golden/hf_nfc_goldens.json samples and seeded
                consonant + sign streams) — verify mode, against the same tokenizer.json with its normalizer removed
                (a temporary copy): on NFC text both give the same ids, so the difference is the verification
  natural       the ASCII natural corpus (workload.natural_corpus), the same pair

Gate: every multilingual prompt accepted by both handles, and identical ids on every prompt verify accepts.  Prints the card's name and power limit with the
numbers.  usage: python scripts/bench_nfc.py [n_prompts] [reps]"""
import json
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import xllm_service_b200 as x  # noqa: E402
from xllm_service_b200 import workload  # noqa: E402

PROMPT = 16384
QWEN2 = os.path.join(ROOT, "tests", "golden", "hf_qwen2_style")


def multilingual_prompts(n, seed=0):
    import make_hf_nfc_fixture as m
    samples = m.nfc_texts() + [" ".join(workload.sentences(4, (8, 20), seed=s)) for s in range(8)]
    samples = [t.encode() for t in samples]
    rnd = random.Random(seed)
    out = []
    for _ in range(n):
        parts, size = [], 0
        while size < PROMPT + 64:
            p = rnd.choice(samples)
            parts.append(p)
            size += len(p) + 1
        b = b" ".join(parts)[:PROMPT]
        out.append(b[:b.rindex(b" ")])       # cut at a space: whole chars, still NFC
    return workload.pack_prompts(out)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers still stand; the report says the limit is unknown
        q = "unknown (%s)" % e
    return name, q


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    tmp = tempfile.mkdtemp(prefix="bench_nfc_")
    with open(os.path.join(QWEN2, "tokenizer.json"), encoding="utf-8") as f:
        tj = json.load(f)
    assert tj["normalizer"] == {"type": "NFC"}
    tj["normalizer"] = None
    with open(os.path.join(tmp, "tokenizer.json"), "w", encoding="utf-8") as f:
        json.dump(tj, f, ensure_ascii=False)
    verify = x.Ingest(tokenizer_path=QWEN2)
    verify.set_nfc_policy(1)
    plain = x.Ingest(tokenizer_path=tmp)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": None, "power_limit, max_sm_clock": None, "prompts": n, "prompt_bytes": PROMPT}
    for name, pb in (("multilingual", multilingual_prompts(n)),
                     ("natural", workload.cut_prompts(workload.natural_corpus(n * PROMPT), PROMPT))):
        m = pb.n
        stride = PROMPT + 16
        d_text = torch.from_numpy(pb.text).cuda()
        d_off = torch.from_numpy(pb.offsets).cuda()
        outs = {}
        for key in ("verify", "plain"):
            outs[key] = (torch.empty((m, stride), dtype=torch.int32, device="cuda"),
                         torch.empty(m, dtype=torch.int32, device="cuda"), torch.empty(m, dtype=torch.int32, device="cuda"))

        def run(key):
            h = verify if key == "verify" else plain
            ids, nid, st = outs[key]
            h.encode_batch_device(m, d_text.data_ptr(), d_off.data_ptr(), ids.data_ptr(), stride, nid.data_ptr(),
                                  st.data_ptr(), stream.cuda_stream)

        times = {"verify": [], "plain": []}
        for key in ("verify", "plain"):   # warm-up: module load, memo tables, scratch
            run(key)
        torch.cuda.synchronize()
        for _ in range(reps):              # alternate the two, same call
            for key in ("verify", "plain"):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run(key)
                e1.record(stream)
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        (iv, nv, sv), (ip, np_, sp) = outs["verify"], outs["plain"]
        ok_status = bool((sv == 0).all().item() and (sp == 0).all().item())
        # ids of the rows verify accepted (all of them, on NFC text) against the handle without a normalizer
        acc = sv == 0
        mask = (torch.arange(stride, device="cuda")[None, :] < nv[:, None]) & acc[:, None]
        same = bool(torch.equal(nv[acc], np_[acc]) and torch.equal(torch.where(mask, iv, 0), torch.where(mask, ip, 0)))
        tv, tp = float(np.median(times["verify"])), float(np.median(times["plain"]))
        result[name] = {"verify_ms": round(tv, 3), "no_normalizer_ms": round(tp, 3),
                        "verify_overhead_pct": round(100 * (tv - tp) / tp, 1),
                        "MB_per_s_verify": round(pb.text.size / tv / 1e3, 1), "text_MB": round(pb.text.size / 1e6, 1),
                        "spread_ms": [round(min(times["verify"]), 3), round(max(times["verify"]), 3),
                                      round(min(times["plain"]), 3), round(max(times["plain"]), 3)],
                        "all_accepted": ok_status, "ids_identical": same,
                        "statuses": {int(k): int(v) for k, v in zip(*np.unique(sv.cpu().numpy(), return_counts=True))}}
        del outs, d_text, d_off
        torch.cuda.empty_cache()
    result["card"], result["power_limit, max_sm_clock"] = card()
    verify.close()
    plain.close()
    print(json.dumps(result))
    gate = result["multilingual"]["all_accepted"] and all(result[k]["ids_identical"] for k in ("multilingual", "natural"))
    sys.exit(0 if gate else 1)


if __name__ == "__main__":
    main()
