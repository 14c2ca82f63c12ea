"""End-to-end parity of xllm_ingest_batch (tokenize -> block hash -> match -> route, chunk-pipelined over
several streams) against the CPU oracle's per-request Scheduler::schedule path."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
import os  # noqa: E402

HERE = os.path.dirname(__file__)
MODEL_DIR = os.path.join(HERE, "golden", "sp_bpe_8k")
NAMES = ["inst%02d" % i for i in range(16)]


def test_pipeline_matches_oracle(oracle):
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    rng = np.random.default_rng(11)
    h = x.Ingest(tokenizer_path=MODEL_DIR, index_capacity=1 << 15)
    h.set_pipeline(37, 1 << 20)  # small chunks: many chunks in flight, odd boundaries
    sp = oracle.SentencePieceOracle(MODEL_DIR)
    P = oracle.PrefixOracle(NAMES)
    vocab = workload.make_vocabulary()
    wb = workload.pack_prompts(vocab)
    _, wcnt = sp.encode_batch(wb.text, wb.offsets, 32)
    T = 1024
    batch, meta = workload.make_prompts_exact_tokens(
        300, T, wcnt, seed=5, shared_prefix=dict(n_prefixes=8, frac=0.8, min_blocks=2, max_blocks=6, block_tokens=128))
    # ragged extras: empty, short, invalid utf-8
    extra = [b"", b"hi", b"\xff\xfe broken \xe6\x97", "日本 語".encode(), b" ".join(vocab[:50])]
    texts = [batch.prompt(i) for i in range(batch.n)] + extra
    b = workload.pack_prompts(texts)
    for i, n in enumerate(NAMES):
        t = 2 if i % 2 else 1
        w, u = int(rng.integers(0, 9)), float(np.float32(rng.random()))
        P.set_instance(n, t)
        P.set_load(n, w, u)
        h.set_instance(i, t)
        h.set_load_metrics(i, w, u)
    # index content: prefixes of the first requests
    ref = oracle.ingest_batch(sp, None, b.text, b.offsets, T)
    for r in range(0, 60):
        keys = oracle.block_hash_chain(ref["ids"][r, :ref["n_ids"][r]])
        i = int(rng.integers(0, len(NAMES)))
        k = keys[:int(rng.integers(0, keys.shape[0] + 1))]
        P.record(NAMES[i], k)
        h.index_apply(i, k)
    P.upload()
    h.index_publish()
    out = h.ingest_batch(b.text, b.offsets, T)
    ref = oracle.ingest_batch(sp, P, b.text, b.offsets, T)
    assert (out["status"] == 0).all()
    assert (out["n_ids"] == ref["n_ids"]).all()
    for r in range(b.n):
        n = ref["n_ids"][r]
        assert (out["ids"][r, :n] == ref["ids"][r, :n]).all(), r
        want = oracle.block_hash_chain(ref["ids"][r, :n])
        assert (out["keys"][r, :want.shape[0]] == want).all(), r
        assert not out["keys"][r, want.shape[0]:].any(), r  # zero padding past the last full block
        m = P.match(ref["ids"][r, :n])
        assert out["match"]["max_matched_block_num"][r] == m["max_matched_block_num"], r
        assert out["match"]["hbm"][r][:len(NAMES)].tolist() == m["hbm"].tolist(), r
        ro = P.route(ref["ids"][r, :n])
        assert bool(out["routing"]["ok"][r]) == ro["ok"]
        assert out["routing"]["prefill_score"][r] == np.float32(ro["prefill_score"]), r
        assert (ro["prefill_argmax"] >> int(out["routing"]["prefill_id"][r])) & 1, r
        assert (ro["decode_argmax"] >> int(out["routing"]["decode_id"][r])) & 1, r
    # tokenizer-only call (no index outputs) and keys-only call
    o2 = h.ingest_batch(b.text, b.offsets, T, want_keys=True, want_match=False)
    assert (o2["ids"] == out["ids"]).all() and (o2["keys"] == out["keys"]).all()
    h.close()


@pytest.mark.parametrize("n_req", [1, 63, 513, 600, 1100, 1537, 4097])
def test_default_pipeline_any_batch_size(oracle, n_req):
    """The default chunk schedule (ramp 512 -> 4096, quarter-size tail) on batch sizes around its break points."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    sp = oracle.SentencePieceOracle(MODEL_DIR)
    texts = [s.encode() for s in workload.sentences(n_req, (1, 12), seed=n_req)]
    b = workload.pack_prompts(texts)
    h = x.Ingest(tokenizer_path=MODEL_DIR)
    try:
        out = h.ingest_batch(b.text, b.offsets, 128, want_match=False)
        chunks, launches = h.last_batch_stats()
        assert chunks >= 1 and launches == 5 * chunks          # encode x3 (express, buffer path, long words) + row prep + hash per chunk
        assert (out["status"] == 0).all()
        ref_ids, ref_n = sp.encode_batch(b.text, b.offsets, 128)
        assert (out["n_ids"] == ref_n).all()
        for r in range(n_req):
            assert (out["ids"][r, :ref_n[r]] == ref_ids[r, :ref_n[r]]).all(), r
    finally:
        h.close()


def test_short_rows_still_get_a_routing_decision(oracle):
    """ids_stride < block_size with match / routing requested: no request has a full block, so the reference's match
    leaves OverlapScores untouched (global_kvcache_mgr.cpp:77-79) and routing takes get_load_metrics' least-loaded
    fallback (instance_mgr.cpp:312-358).  The batch call must return exactly that — zeroed match rows and a real
    decision — not whatever the output buffers held before."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    h = x.Ingest(tokenizer_path=MODEL_DIR, index_capacity=1024)
    P = oracle.PrefixOracle(NAMES)
    for i, n in enumerate(NAMES):
        t = 2 if i % 2 else 1
        P.set_instance(n, t)
        P.set_load(n, i % 5, (i * 7 % 16) / 16.0)
        h.set_instance(i, t)
        h.set_load_metrics(i, i % 5, (i * 7 % 16) / 16.0)
    texts = [s.encode() for s in workload.sentences(50, (1, 8), seed=3)] + [b""]
    b = workload.pack_prompts(texts)
    n = b.n
    ids = np.zeros((n, 64), np.int32)
    n_ids = np.zeros(n, np.int32)
    status = np.zeros(n, np.int32)
    match = np.full(n, 0xAB, dtype=np.uint8).repeat(400).view(x._lib.MATCH_DTYPE)    # poisoned output buffers
    routing = np.full(n * 20, 0xCD, dtype=np.uint8).view(x._lib.ROUTING_DTYPE)
    h.ingest_batch_ptrs(n, b.text.ctypes.data, b.offsets.ctypes.data, ids.ctypes.data, 64, n_ids.ctypes.data,
                        status.ctypes.data, 0, 0, match.ctypes.data, routing.ctypes.data)
    chunks, launches = h.last_batch_stats()
    assert launches == 5 * chunks      # encode x3 + row prep + match/route, no hash
    want = P.route(np.zeros(0, np.int32))
    assert want["ok"]
    for r in range(n):
        assert match["max_block_num"][r] == 0 and match["max_matched_block_num"][r] == 0 and match["instances"][r] == 0
        assert not match["hbm"][r].any() and not match["dram"][r].any() and not match["ssd"][r].any()
        assert routing["ok"][r] == 1
        assert routing["prefill_score"][r] == np.float32(want["prefill_score"])
        assert (want["prefill_argmax"] >> int(routing["prefill_id"][r])) & 1
        assert (want["decode_argmax"] >> int(routing["decode_id"][r])) & 1
    h.close()


def test_narrow_id_download_equals_int32(oracle):
    """xllm_ingest_io::ids_u16: the same batch with uint16 ids — every other output identical, ids equal after
    widening; refused for a vocabulary that does not fit 16 bits."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    texts = [s.encode() for s in workload.sentences(700, (1, 90), seed=8)] + [b"", "日本語 text".encode()]
    b = workload.pack_prompts(texts)
    h = x.Ingest(tokenizer_path=MODEL_DIR, index_capacity=1024)
    h.set_pipeline(53, 1 << 20)
    h.set_instance(0, 1)
    h.set_instance(1, 2)
    h.set_load_metrics(0, 1, 0.5)
    h.set_load_metrics(1, 2, 0.25)
    a = h.ingest_batch(b.text, b.offsets, 200)
    c = h.ingest_batch(b.text, b.offsets, 200, ids_u16=True)
    assert c["ids"].dtype == np.uint16
    valid = np.arange(200)[None, :] < np.minimum(a["n_ids"], 200)[:, None]
    assert (a["ids"][valid] == c["ids"][valid]).all()
    for f in ("n_ids", "status", "keys"):
        assert (a[f] == c[f]).all(), f
    assert a["match"].tobytes() == c["match"].tobytes() and a["routing"].tobytes() == c["routing"].tobytes()
    h.close()
    os.environ["XLLM_SP_FORCE_WIDE"] = "1"      # kernels built for > 16-bit ids keep working with the narrow download
    try:
        hw = x.Ingest(tokenizer_path=MODEL_DIR)
        d = hw.ingest_batch(b.text, b.offsets, 200, want_match=False, ids_u16=True)
        assert (d["ids"][valid] == a["ids"][valid]).all()
        hw.close()
    finally:
        del os.environ["XLLM_SP_FORCE_WIDE"]
    # 128 471 entries: ids past 65 535 cannot be downloaded as uint16
    hb = x.Ingest(tokenizer_path=os.path.join(HERE, "golden", "hf_natural_128k"))
    try:
        with pytest.raises(x.IngestError) as e:
            hb.ingest_batch(b.text, b.offsets, 200, want_match=False, ids_u16=True)
        assert e.value.code == -5      # XLLM_ERR_UNSUPPORTED
    finally:
        hb.close()
