"""Exact NFC verification on the device (csrc/hf_nfc.cu, xllm_set_nfc_policy(h, XLLM_NFC_VERIFY)) for the Qwen2-style
tokenizer.json (`normalizer: NFC`): statuses against the Python restatement of the rule (tests/nfc_oracle.py), ids
against the pip-`tokenizers` goldens (tests/golden/make_hf_nfc_fixture.py) and the CPU oracle, through every entry
point that tokenises, and the default policy left as it was."""
import ctypes
import json
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import nfc_oracle  # noqa: E402

QWEN2 = os.path.join(HERE, "golden", "hf_qwen2_style")
LLAMA3 = os.path.join(HERE, "golden", "hf_llama3_style")
GOLD = os.path.join(HERE, "golden", "hf_nfc_goldens.json")
STATUS_OF = {0: 0, 1: -5, 2: -1}
VERIFY = 1


def _gold():
    with open(GOLD) as f:
        return json.load(f)["cases"]


def _handle(path=QWEN2, verify=True):
    import xllm_service_b200 as x
    h = x.Ingest(tokenizer_path=path)
    if verify:
        h.set_nfc_policy(VERIFY)
    return h


def _encode(h, texts, stride=None):
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    stride = stride or max(16, max((len(t) for t in texts), default=0) + 8)
    ids, n_ids, status = h.encode_batch(b.text, b.offsets, stride)
    return [ids[i, :n_ids[i]].tolist() for i in range(len(texts))], status, n_ids


def _check_vs_oracle(texts, got, status, n_ids, hf):
    for i, t in enumerate(texts):
        want = STATUS_OF[nfc_oracle.nfc_verdict(t)]
        if want == 0 and status[i] == -6:     # a single pre-token longer than the device scratch: not this feature's
            continue
        assert status[i] == want, (i, len(t), t[:40])
        if want == 0:
            assert got[i] == hf.prefix_ids + hf.encode(t).tolist() + hf.suffix_ids, (i, len(t), t[:40])
        else:
            assert n_ids[i] == 0, i


@pytest.fixture(scope="module")
def qwen(oracle):
    h = _handle()
    yield h, oracle.HfBpeOracle(QWEN2)
    h.close()


def test_goldens(qwen):
    h, _ = qwen
    g = _gold()
    texts = [bytes.fromhex(c["text"]) for c in g["nfc"]]
    got, status, _ = _encode(h, texts)
    assert (status == 0).all(), [(texts[i][:30], int(status[i])) for i in np.nonzero(status)[0][:5]]
    assert got == [c["ids"] for c in g["nfc"]]
    refused = [bytes.fromhex(c["text"]) for c in g["not_nfc"] + g["wheel_older"]]
    _, status, n_ids = _encode(h, refused)
    assert (status == -5).all() and (n_ids == 0).all(), status.tolist()


def test_fuzz_vs_oracle(qwen):
    h, hf = qwen
    rnd = random.Random(41)
    texts = []
    for i in range(20_000):
        s = "".join(rnd.choice(nfc_oracle.FUZZ_ALPHABET) for _ in range(rnd.randrange(0, 40)))
        b = s.encode()
        if i % 50 == 0 and b:               # now and then a malformed byte somewhere
            k = rnd.randrange(len(b) + 1)
            b = b[:k] + rnd.choice((b"\xff", b"\x80", b"\xc3", b"\xed\xa0\x80")) + b[k:]
        texts.append(b)
    got, status, n_ids = _encode(h, texts)
    assert (status == 0).sum() > 2000 and (status == -5).sum() > 4000 and (status == -1).sum() > 100
    _check_vs_oracle(texts, got, status, n_ids, hf)


def test_long_texts_cross_windows_and_the_staging_buffer(qwen):
    """3 .. 40 KB of mixed scripts: Maybe chunks straddle the 512-byte verify windows (the chunk start is found by
    reading back across them) and the 2 KB staging buffer of the tokenizer kernels."""
    h, hf = qwen
    g = _gold()
    samples = [bytes.fromhex(c["text"]).decode() for c in g["nfc"]]
    rnd = random.Random(5)
    texts = []
    for k in range(60):
        parts, n = [], 0
        goal = rnd.randrange(3000, 40000)
        while n < goal:
            p = rnd.choice(samples) + " " + "ab " * rnd.randrange(0, 200)
            parts.append(p)
            n += len(p.encode())
        texts.append("".join(parts).encode())
    for pad in range(490, 530):              # a Bengali / Tamil / Hangul Maybe chunk at every offset of a window seam
        texts.append(("a" * pad + "\u0995\u09be\u0bca \uac01 x" + "\u0301" * 20).encode())
        texts.append(("a" * pad + "\u1100\u1161 and \u0b95\u0bca").encode())   # Hangul L+V: not NFC
    for pad in range(2030, 2060):
        texts.append(("ab " * (pad // 3) + "\u0929\u0915\u093c\u0940 \u0915\u094d\u0937 \u0ddc").encode())
    got, status, n_ids = _encode(h, texts)
    assert (status == 0).sum() > 100 and (status == -5).sum() == 40
    _check_vs_oracle(texts, got, status, n_ids, hf)


def test_chunk_cap_and_long_mark_runs(qwen):
    h, hf = qwen
    texts = []
    for pad in (0, 3, 500, 511, 2040):    # the chunk at both sides of a verify window / staging buffer seam
        lead = "ab " * (pad // 3) + "a" * (pad % 3)
        texts.append((lead + " x" + "\u0301" * 31 + " y").encode())     # 32 code points: accepted
        texts.append((lead + " x" + "\u0301" * 32 + " y").encode())     # 33: refused although in NFC
    texts.append(("x" + "\u0301" * 10_000).encode())                           # 10 K Maybe marks: refused
    texts.append(("x" + "\u0316" * 10_000).encode())                           # no Maybe char: no cap
    texts.append((" x\u0316" * 5000).encode())
    got, status, n_ids = _encode(h, texts)
    assert status[:10].tolist() == [0, -5] * 5
    assert status[10] == -5 and status[11] in (0, -6) and status[12] == 0
    for i in (0, 2, 4, 6, 8, 12):
        assert got[i] == hf.prefix_ids + hf.encode(texts[i]).tolist() + hf.suffix_ids


def test_malformed_utf8_wins(qwen):
    h, _ = qwen
    texts = [b"e\xcc\x81\xff", b"\xff\xe2\x84\xab", b"\xe2\x84\xab" + b"a" * 3000 + b"\xc3",
             "\u0958".encode() + b"\xed\xa0\x80", b"ok \xe0\xa4\x95\xe0\xa4\xbc \xf4\x90\x80\x80"]
    _, status, n_ids = _encode(h, texts)
    assert status.tolist() == [-1] * 5 and (n_ids == 0).all()


def test_every_scalar_value_in_context(qwen):
    h, _ = qwen
    cps = [cp for cp in range(0x110000) if not 0xD800 <= cp < 0xE000]
    for pre, post in (("", ""), ("x", "\u0301"), ("\u1100", ""), ("a\u0316", "\u0300")):
        texts = [(pre + chr(cp) + post).encode() for cp in cps]
        _, status, _ = _encode(h, texts, stride=16)
        want = np.array([STATUS_OF[nfc_oracle.nfc_verdict(t)] for t in texts], np.int32)
        bad = np.nonzero(status != want)[0]
        assert bad.size == 0, [(hex(cps[i]), int(status[i]), int(want[i])) for i in bad[:10]]


def _mixed_texts():
    g = _gold()
    texts = [bytes.fromhex(c["text"]) for c in g["nfc"]] + [bytes.fromhex(c["text"]) for c in g["not_nfc"]]
    rnd = random.Random(9)
    texts += ["".join(rnd.choice(nfc_oracle.FUZZ_ALPHABET) for _ in range(rnd.randrange(0, 30))).encode()
              for _ in range(3000)]
    return texts


def test_ingest_batch_segments_device_pointer_and_clone(qwen):
    import torch
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    h, _ = qwen
    texts = _mixed_texts()
    ref, ref_st, ref_n = _encode(h, texts, stride=512)
    # xllm_ingest_batch over several pipeline chunks
    b = workload.pack_prompts(texts)
    h.set_pipeline(400, 1 << 20)
    out = h.ingest_batch(b.text, b.offsets, 512, want_keys=False, want_match=False)
    chunks, launches = h.last_batch_stats()
    assert chunks > 3 and launches == 3 * chunks                # verify + buffer path + long words
    assert out["status"].tolist() == ref_st.tolist()
    for i in np.nonzero(ref_st == 0)[0]:
        assert out["ids"][i, :out["n_ids"][i]].tolist() == ref[i]
    # xllm_ingest_batch_segments: a piece that is not NFC fails only its request
    pieces = [b"fine", "\u0995\u09be".encode(), "e\u0301".encode(), "\u0e01\u0e48 ok".encode(), b"tail"]
    pb = workload.pack_prompts(pieces)
    sb = workload.SegmentBatch(pb.text, pb.offsets, np.array([0, 2, 4, 6], np.int32),
                               np.array([-1, -1, -1, 3, -1, -1], np.int32), np.arange(3, dtype=np.int32),
                               np.zeros(3, bool), np.zeros(3, np.int32))
    so = h.ingest_batch_segments(sb, 64, want_match=False)
    assert so["status"].tolist() == [0, -5, 0] and so["n_ids"][1] == 0
    # the device-pointer entry
    dev = torch.device("cuda")
    d_text = torch.from_numpy(b.text.copy()).to(dev)
    d_off = torch.from_numpy(b.offsets.copy()).to(dev)
    n = len(texts)
    d_ids = torch.zeros((n, 512), dtype=torch.int32, device=dev)
    d_n = torch.zeros(n, dtype=torch.int32, device=dev)
    d_st = torch.full((n,), -9, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    h.encode_batch_device(n, d_text.data_ptr(), d_off.data_ptr(), d_ids.data_ptr(), 512, d_n.data_ptr(),
                          d_st.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert d_st.cpu().numpy().tolist() == ref_st.tolist()
    ids_d, n_d = d_ids.cpu().numpy(), d_n.cpu().numpy()
    for i in np.nonzero(ref_st == 0)[0]:
        assert ids_d[i, :n_d[i]].tolist() == ref[i]
    # a clone keeps the policy
    c = ctypes.c_void_p()
    x._lib.check(h._L.xllm_ingest_clone(h._h, ctypes.byref(c)))
    w = x.Ingest.__new__(x.Ingest)
    w._L, w._h, w.block_size, w.seed = h._L, c, 128, 1024
    try:
        got, st, _ = _encode(w, texts, stride=512)
        assert st.tolist() == ref_st.tolist() and got == ref
    finally:
        w.close()


def test_default_policy_is_unchanged(oracle):
    from xllm_service_b200 import workload
    # Thai in NFC with a vowel sign and tone marks (ccc 103 / 107): refused by the inert-char proof
    thai = "\u0e1c\u0e39\u0e49\u0e04\u0e19 \u0e20\u0e32\u0e29\u0e32\u0e44\u0e17\u0e22 \u0e19\u0e49\u0e33".encode()
    h = _handle(verify=False)
    try:
        _, status, _ = _encode(h, [thai, b"plain", "x\u0301".encode()])
        assert status.tolist() == [-5, 0, -5]
        with pytest.raises(Exception):
            h.set_nfc_policy(2)
        texts = [s.encode() for s in workload.sentences(1100, (1, 12), seed=4)]
        b = workload.pack_prompts(texts)
        h.set_pipeline(256, 1 << 20)
        h.ingest_batch(b.text, b.offsets, 128, want_match=False)
        chunks, launches = h.last_batch_stats()
        assert chunks > 1 and launches == (2 + 2) * chunks     # buffer path + long words, + row prep + hash
        h.set_nfc_policy(VERIFY)
        h.ingest_batch(b.text, b.offsets, 128, want_match=False)
        assert h.last_batch_stats() == (chunks, (3 + 2) * chunks)
        h.set_nfc_policy(0)
        _, status, _ = _encode(h, [thai])
        assert status.tolist() == [-5]
    finally:
        h.close()
    # XLLM_HF_NFC_VERIFY=1 sets the policy at create
    os.environ["XLLM_HF_NFC_VERIFY"] = "1"
    try:
        h = _handle(verify=False)
    finally:
        os.environ.pop("XLLM_HF_NFC_VERIFY")
    try:
        _, status, _ = _encode(h, [thai])
        assert status.tolist() == [0]
    finally:
        h.close()


def test_no_effect_without_the_nfc_normalizer(oracle):
    texts = _mixed_texts()
    a, b = _handle(LLAMA3, verify=False), _handle(LLAMA3, verify=True)
    try:
        ga, sa, _ = _encode(a, texts)
        gb, sb, _ = _encode(b, texts)
        assert (sa == 0).all() and sa.tolist() == sb.tolist() and ga == gb
    finally:
        a.close()
        b.close()


def test_ingest_batcher_serves_marks_on_the_device(oracle, tmp_path):
    """host/ingest_batcher.h sets XLLM_NFC_VERIFY: Thai and Hindi in NFC come back from the device, a decomposed text
    is still refused (tests/cpp/batcher_main.cc)."""
    texts = [b"plain ascii first", "\u0e1c\u0e39\u0e49\u0e04\u0e19 \u0e20\u0e32\u0e29\u0e32\u0e44\u0e17\u0e22 \u0e19\u0e49\u0e33".encode(),
             "\u0928\u0939\u0940\u0902 \u0915\u093c\u0932\u092e \u0939\u093f\u0902\u0926\u0940".encode(),
             "cafe\u0301".encode(), "\u0995\u09be\u0997\u099c".encode()]
    pf = tmp_path / "prompts.bin"
    with open(pf, "wb") as f:
        for t in texts:
            f.write(struct.pack("<I", len(t)) + t)
    exe = tmp_path / "batcher_main"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "xllm_service_b200", "host"),
                           os.path.join(HERE, "cpp", "batcher_main.cc"), "-o", str(exe),
                           "-L", os.path.join(ROOT, "xllm_service_b200"), "-lxllm_ingest",
                           "-Wl,-rpath," + os.path.join(ROOT, "xllm_service_b200")])
    p = subprocess.run([str(exe), QWEN2, str(pf), "4", "8", "200"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr
    hf = oracle.HfBpeOracle(QWEN2)
    lines = [[int(v) for v in line.split()] for line in p.stdout.strip().split("\n")]
    assert [f[0] for f in lines] == [0, 0, 0, -5, 0]
    for t, f in zip(texts, lines):
        if f[0] == 0:
            assert f[4:] == hf.prefix_ids + hf.encode(t).tolist() + hf.suffix_ids
