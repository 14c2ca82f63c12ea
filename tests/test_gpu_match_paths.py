"""Block keys, prefix match and routing away from the configuration bench.py runs, against the CPU oracle:
  * the whole batch path (prep_rows_kernel, the generic hash kernel, match_route_kernel) at block sizes other than 128,
    with truncated rows, an explicit keys_stride, segmented requests and 1 / 2 pipeline slots;
  * long requests through match_route_kernel: first misses at every lane of the first, a middle and the last probe
    wave, tier-only hits, entries with three empty masks, 65 535 blocks;
  * the 65 535-block limit of the 16-bit scores of xllm_match_out on the batch path;
  * the device-pointer entry points on a caller's stream (encode -> hash -> match, and the split probe / score pair);
  * the bulk-copy variant of the 128-token hash kernel (XLLM_XXH3_BULK=1), in a child process.
Match rows are compared in full (max_block_num, max_matched_block_num, instances, the three score maps of all 64 ids);
routing must agree on ok and on the float32 scores, and its choices must lie in the oracle's arg-max sets."""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SP_DIR = os.path.join(HERE, "golden", "sp_bpe_8k")
HF_DIR = os.path.join(HERE, "golden", "hf_llama3_style")
NAMES = ["node-%02d" % i for i in range(64)]
SEED = 1024
BLOCK_SIZES = [1, 2, 16, 31, 64, 100, 127, 129, 251]


# ----------------------------------------------------------------------------------------------------------- helpers
def _check_match_route(P, tokens, mrow, rrow, where):
    """One request's device match / routing row against GlobalKVCacheMgr::match + CacheAwareRouting on `tokens`."""
    m = P.match(tokens)
    assert mrow["max_block_num"] == m["max_block_num"], where
    assert mrow["max_matched_block_num"] == m["max_matched_block_num"], where
    assert mrow["instances"] == m["instances"], where
    for tier in ("hbm", "dram", "ssd"):
        assert mrow[tier].tolist() == m[tier].tolist(), (where, tier)
    ro = P.route(tokens)
    assert bool(rrow["ok"]) == ro["ok"], where
    if not ro["ok"]:
        return
    assert rrow["prefill_score"] == np.float32(ro["prefill_score"]), where
    pid = int(rrow["prefill_id"])
    if ro["prefill_argmax"] == 0:
        assert pid == -1, where
    else:
        assert pid >= 0 and (ro["prefill_argmax"] >> pid) & 1, (where, pid, ro)
    did = int(rrow["decode_id"])
    if ro["decode_id"] == -1 and ro["decode_argmax"] == 0:
        assert did == -1, where
    else:
        assert rrow["decode_score"] == np.float32(ro["decode_score"]), where
        assert did >= 0 and (ro["decode_argmax"] >> did) & 1, (where, did, ro)


def _view(rng):
    """64 instances: default / prefill / decode / mix, some not schedulable, some never given load metrics."""
    view = []
    for _ in range(64):
        t = int(rng.choice([0, 1, 2, 2, 3]))
        sched = bool(rng.random() > 0.15)
        load = (int(rng.integers(0, 6)), float(np.float32(rng.random()))) if rng.random() > 0.2 else None
        view.append((t, sched, load))
    return view


def _set_view(view, h=None, P=None):
    for i, (t, sched, load) in enumerate(view):
        if h is not None:
            h.set_instance(i, t, sched)
            if load:
                h.set_load_metrics(i, *load)
        if P is not None:
            P.set_instance(NAMES[i], t, sched)
            if load:
                P.set_load(NAMES[i], *load)


def _events(key_rows, rng, windows=2, per_window=60):
    """stored / offload / removed events drawn from real key chains, `None` = publish."""
    key_rows = [k for k in key_rows if k.shape[0]]
    ev = []
    for _ in range(windows):
        for _ in range(per_window):
            i = int(rng.integers(0, 64))
            kb = key_rows[int(rng.integers(0, len(key_rows)))]
            upto = int(rng.integers(1, kb.shape[0] + 1))
            s = kb[:upto] if rng.random() < 0.7 else kb[rng.integers(0, kb.shape[0], size=int(rng.integers(0, 20)))]
            o = kb[rng.integers(0, kb.shape[0], size=int(rng.integers(0, 6)))]
            r = kb[rng.integers(0, kb.shape[0], size=int(rng.integers(0, 3)))]
            ev.append((i, s, o, r))
        ev.append(None)
    return ev


def _apply(ev, h=None, P=None):
    for e in ev:
        if e is None:
            if h is not None:
                h.index_publish()
            if P is not None:
                P.upload()
        else:
            if h is not None:
                h.index_apply(*e)
            if P is not None:
                P.record(NAMES[e[0]], e[1], e[2], e[3])


def _handle(env=None, **kw):
    """Ingest handle created with `env` set (XLLM_PIPE_SLOTS is read at create), the environment restored after."""
    import xllm_service_b200 as x
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return x.Ingest(**kw)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@functools.lru_cache(maxsize=None)
def _word_counts():
    from oracle import oracle as o
    from xllm_service_b200 import workload
    sp = o.SentencePieceOracle(SP_DIR)
    wb = workload.pack_prompts(workload.make_vocabulary())
    _, wcnt = sp.encode_batch(wb.text, wb.offsets, 32)
    return wcnt


def _tokens_for(bs):
    return max(1024, 12 * bs)


@functools.lru_cache(maxsize=None)
def _batch(bs):
    """~300 prompts of exactly T tokens sharing prefixes of whole bs-token blocks, then ragged extras: an empty
    prompt, fewer ids than one block, k*bs - 1, k*bs and k*bs + 1 ids.  Returns (PromptBatch, T, extra lengths)."""
    from xllm_service_b200 import workload
    T = _tokens_for(bs)
    nb = T // bs
    wcnt = _word_counts()
    shared = dict(n_prefixes=8, frac=0.8, min_blocks=max(1, nb // 8), max_blocks=max(2, nb // 2), block_tokens=bs)
    batch, _ = workload.make_prompts_exact_tokens(300, T, wcnt, seed=bs, shared_prefix=shared)
    texts = [batch.prompt(i) for i in range(batch.n)] + [b""]
    k = max(1, nb // 2)
    lens = ([bs - 1] if bs > 1 else []) + [k * bs - 1, k * bs, k * bs + 1]
    extra = [0]
    for n_tok in lens:
        eb, _ = workload.make_prompts_exact_tokens(2, n_tok, wcnt, seed=bs, shared_prefix=shared)
        texts += [eb.prompt(i) for i in range(eb.n)]
        extra += [n_tok, n_tok]
    return workload.pack_prompts(texts), T, extra


def _setup_batch(oracle, bs, env=None):
    """Handle + oracle with the 64-instance view and index content from the batch's own key chains."""
    import xllm_service_b200 as x  # noqa: F401
    b, T, extra = _batch(bs)
    sp = oracle.SentencePieceOracle(SP_DIR)
    ref = oracle.ingest_batch(sp, None, b.text, b.offsets, T, n_threads=os.cpu_count() or 1)
    rng = np.random.default_rng(100 + bs)
    view = _view(rng)
    key_rows = [oracle.block_hash_chain(ref["ids"][r, :ref["n_ids"][r]], bs, SEED) for r in range(80)]
    ev = _events(key_rows, rng)
    h = _handle(env, tokenizer_path=SP_DIR, block_size=bs, xxh3_seed=SEED, index_capacity=1 << 18)
    h.set_pipeline(37, 1 << 20)       # small odd chunks: many chunks in flight, odd boundaries
    P = oracle.PrefixOracle(NAMES, bs, SEED)
    _set_view(view, h, P)
    _apply(ev, h, P)
    assert h.index_size() == P.size()
    return h, P, b, T, extra, ref


def _ingest_raw(h, b, ids_stride, keys_stride):
    """xllm_ingest_batch with an explicit keys_stride."""
    import xllm_service_b200 as x
    n = b.n
    out = {"ids": np.zeros((n, ids_stride), np.int32), "n_ids": np.zeros(n, np.int32), "status": np.zeros(n, np.int32),
           "keys": np.zeros((n, keys_stride, 16), np.uint8), "match": np.zeros(n, x._lib.MATCH_DTYPE),
           "routing": np.zeros(n, x._lib.ROUTING_DTYPE)}
    h.ingest_batch_ptrs(n, b.text.ctypes.data, b.offsets.ctypes.data, out["ids"].ctypes.data, ids_stride,
                        out["n_ids"].ctypes.data, out["status"].ctypes.data, out["keys"].ctypes.data, keys_stride,
                        out["match"].ctypes.data, out["routing"].ctypes.data)
    return out


def _check_batch(oracle, P, out, ref, bs, ids_stride, keys_stride=None):
    """Every row of an ingest_batch result against the oracle: a truncated row hashes and matches the ids that were
    written (ids[:ids_stride]); an explicit keys_stride caps the hashed and matched blocks."""
    for r in range(ref["n_ids"].size):
        n = int(ref["n_ids"][r])
        full = ref["ids"][r, :n]
        have = min(n, ids_stride)
        assert out["n_ids"][r] == n, r
        assert out["status"][r] == (1 if n > ids_stride else 0), r
        assert (out["ids"][r, :have] == full[:have]).all(), r
        seen = full[:have] if keys_stride is None else full[:min(have, keys_stride * bs)]
        want = oracle.block_hash_chain(seen, bs, SEED)
        assert (out["keys"][r, :want.shape[0]] == want).all(), r
        assert not out["keys"][r, want.shape[0]:].any(), r      # zero padding past the last full block
        _check_match_route(P, seen, out["match"][r], out["routing"][r], (bs, ids_stride, keys_stride, r))


# ---------------------------------------------------------------- A. the batch path at other block sizes
@pytest.mark.parametrize("bs", BLOCK_SIZES)
def test_batch_path_at_block_size(oracle, bs):
    h, P, b, T, extra, ref = _setup_batch(oracle, bs)
    try:
        # the ragged extras really have the lengths they were built for
        assert ref["n_ids"][-len(extra):].tolist() == extra
        out = h.ingest_batch(b.text, b.offsets, T)
        _check_batch(oracle, P, out, ref, bs, T)
        m = out["match"]
        assert (m["max_matched_block_num"] > 0).sum() > 50, "the index content must produce real prefix matches"
        # truncated rows: an ids_stride that is not a multiple of bs, full-length rows longer than it (status 1)
        s = T * 2 // 3
        while bs > 1 and s % bs == 0:
            s -= 1
        out = h.ingest_batch(b.text, b.offsets, s)
        assert (out["status"] == 1).sum() >= 300
        _check_batch(oracle, P, out, ref, bs, s)
        # an explicit keys_stride below ids_stride / bs: keys and match cover exactly the first keys_stride blocks
        ks = max(1, (T // bs) // 3)
        assert ks < T // bs
        out = _ingest_raw(h, b, T, ks)
        _check_batch(oracle, P, out, ref, bs, T, keys_stride=ks)
    finally:
        h.close()


def test_pipe_slots_do_not_change_results(oracle):
    """XLLM_PIPE_SLOTS=1 / 2: every chunk waits for the download of the chunk that last held its slot's buffers before
    reusing them.  All outputs byte-identical to the default (4 slots) handle's; ids up to each row's n_ids (the rest
    of a row is not written)."""
    bs = 16
    outs = []
    for env in ({}, {"XLLM_PIPE_SLOTS": "1"}, {"XLLM_PIPE_SLOTS": "2"}):
        h, P, b, T, _, _ = _setup_batch(oracle, bs, env)
        try:
            outs.append(h.ingest_batch(b.text, b.offsets, T))
            chunks, _ = h.last_batch_stats()
            assert chunks > 4
        finally:
            h.close()
    written = np.arange(T)[None, :] < np.minimum(outs[0]["n_ids"], T)[:, None]
    for o in outs[1:]:
        assert np.array_equal(o["ids"][written], outs[0]["ids"][written])
        for f in ("n_ids", "status", "keys", "match", "routing"):
            assert np.array_equal(o[f].view(np.uint8), outs[0][f].view(np.uint8)), f


def _oracle_ids(encode_piece, b, r):
    """concatenation of per-piece encodes and id spans of request r"""
    piece_of_seg = np.cumsum(b.seg_len < 0) - (b.seg_len < 0)
    span_of_seg = np.cumsum(np.maximum(b.seg_len, 0)) - np.maximum(b.seg_len, 0)
    out = []
    for s in range(b.req_seg_start[r], b.req_seg_start[r + 1]):
        ln = int(b.seg_len[s])
        if ln < 0:
            p = piece_of_seg[s]
            out.extend(encode_piece(b.text[b.offsets[p]:b.offsets[p + 1]].tobytes()))
        else:
            out.extend(b.span_ids[span_of_seg[s]:span_of_seg[s] + ln].tolist())
    return np.asarray(out, np.int32)


def test_segmented_batch_at_block_size_16(oracle):
    """xllm_ingest_batch_segments on the HF backend (template ids per text piece) with 16-token blocks."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    bs = 16
    rng = np.random.default_rng(16)
    H = oracle.HfBpeOracle(HF_DIR)

    def enc(t):
        return H.prefix_ids + H.encode(t).tolist() + H.suffix_ids

    b = workload.make_c5_batch(120, _word_counts(), seed=16, min_tokens=16, max_tokens=3000,
                               shared_prefix=dict(n_prefixes=6, frac=0.6, min_blocks=2, max_blocks=40, block_tokens=bs))
    assert (b.seg_len >= 0).sum() > 10
    want = [_oracle_ids(enc, b, r) for r in range(b.n)]
    T = 8192
    assert max(w.size for w in want) < T
    h = x.Ingest(tokenizer_path=HF_DIR, block_size=bs, xxh3_seed=SEED, index_capacity=1 << 16)
    h.set_pipeline(41, 1 << 20)
    P = oracle.PrefixOracle(NAMES, bs, SEED)
    try:
        _set_view(_view(rng), h, P)
        _apply(_events([oracle.block_hash_chain(w, bs, SEED) for w in want[::2]], rng), h, P)
        out = h.ingest_batch_segments(b, T)
        assert (out["status"] == 0).all()
        for r in range(b.n):
            n = want[r].size
            assert out["n_ids"][r] == n, r
            assert (out["ids"][r, :n] == want[r]).all(), r
            keys = oracle.block_hash_chain(want[r], bs, SEED)
            assert (out["keys"][r, :keys.shape[0]] == keys).all(), r
            assert not out["keys"][r, keys.shape[0]:].any(), r
            _check_match_route(P, want[r], out["match"][r], out["routing"][r], r)
        assert (out["match"]["max_matched_block_num"] > 32).any()
    finally:
        h.close()


# ------------------------------------------------------------------ B. long requests through match_route_kernel
def test_long_requests_every_first_miss_lane(oracle):
    """Block size 1: n tokens give n keys.  A base sequence of 65 535 blocks whose every block is held by instances 0
    and 63 (63 in HBM on the last block, so its HBM score is 65 535) plus ~8 % of the others; one block in ten is held
    in HBM only, in DRAM only or in SSD only.  Requests: prefixes of every length around the 32-block waves, and 4 096
    blocks with the first miss at every lane of the first, a middle and the last wave.  A second sequence holds an
    entry whose three masks are empty (a miss) in front of entries that would match."""
    import xllm_service_b200 as x
    rng = np.random.default_rng(65535)
    L = 65535
    base = rng.integers(-2**31, 2**31, size=L, dtype=np.int64).astype(np.int32)
    K = oracle.block_hash_chain(base, 1, SEED)
    cls = rng.choice(4, size=L, p=[0.7, 0.1, 0.1, 0.1])     # 0 mixed, 1 HBM only, 2 DRAM only, 3 SSD only
    cls[-1] = 0
    tier = np.where(cls == 0, rng.integers(1, 4, size=(64, L)), cls[None, :])   # 1 HBM, 2 DRAM, 3 SSD
    state = np.where(rng.random((64, L)) < 0.08, tier, 0)
    state[0] = tier[0]
    state[63] = np.where(cls == 0, 1, cls)
    h = x.Ingest(block_size=1, xxh3_seed=SEED, index_capacity=1 << 17)
    P = oracle.PrefixOracle(NAMES, 1, SEED)
    try:
        _set_view(_view(rng), h, P)
        for i in range(64):
            stored, off1, off2 = K[state[i] > 0], K[state[i] >= 2], K[state[i] == 3]
            h.index_apply(i, stored=stored, offload=off1)      # HBM -> DRAM
            P.record(NAMES[i], stored, off1)
            h.index_apply(i, offload=off2)                      # DRAM -> SSD
            P.record(NAMES[i], (), off2)
        B2 = rng.integers(0, 152000, size=4096).astype(np.int32)
        K2 = oracle.block_hash_chain(B2, 1, SEED)
        h.index_apply(40, stored=K2)
        P.record(NAMES[40], K2)
        h.index_publish()
        P.upload()
        hole = 1500                                             # replica PUT of an entry with three empty masks
        h.index_put(K2[hole], 0, 0, 0)
        P.put(K2[hole])
        h.index_publish()
        for k in (K[5], K[L - 1], K2[hole - 1]):
            assert h.index_get(k) == P.get(k)

        reqs = [base[:n] for n in (0, 1, 31, 32, 33, 63, 64, 65, 96, 97, 1000, 4096, 65535)]
        for wave in (0, 64, 127):                               # first, a middle and the last wave of 4 096 blocks
            for lane in range(32):
                t = base[:4096].copy()
                t[wave * 32 + lane] ^= 1
                reqs.append(t)
        reqs += [B2[:hole], B2[:hole + 1], B2]
        keys = [oracle.block_hash_chain(t, 1, SEED) for t in reqs]
        n_blocks = np.array([k.shape[0] for k in keys], np.int32)
        key_start = np.zeros(len(keys), np.int64)
        np.cumsum(n_blocks[:-1], out=key_start[1:])
        match, routing = h.match_route(np.concatenate(keys), key_start, n_blocks)
        for r, t in enumerate(reqs):
            _check_match_route(P, t, match[r], routing[r], (r, t.size))
        full = 13 - 1
        assert match["max_matched_block_num"][full] == L and match["hbm"][full][63] == L
        miss = match["max_matched_block_num"][13:13 + 96]
        assert miss.tolist() == [w * 32 + l for w in (0, 64, 127) for l in range(32)]
        assert match["max_matched_block_num"][-3:].tolist() == [hole, hole, hole]
        # tier-only blocks: DRAM / SSD scores deep in the request, in both halves of the lanes' instance pairs
        for tier in ("dram", "ssd"):
            assert (match[tier][full][:32] > 60000).sum() > 10 and (match[tier][full][32:] > 60000).sum() > 10
    finally:
        h.close()


# ------------------------------------------------------------- C. the 65 535-block limit on the batch path
def test_batch_refuses_rows_of_more_than_65535_blocks(oracle):
    """xllm_match_out keeps scores as uint16 (1 + the last matched block): a row of 65 536 blocks would report 0, as if
    the instance holding every block were absent.  With match / routing requested the batch is refused; at 65 535
    blocks it equals the oracle; a keys-only batch has no such limit."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    batch, _ = workload.make_prompts_exact_tokens(1, 65536, _word_counts(), seed=3)
    sp = oracle.SentencePieceOracle(SP_DIR)
    ids = sp.encode(batch.prompt(0))
    assert ids.size == 65536
    keys = oracle.block_hash_chain(ids, 1, SEED)
    h = x.Ingest(tokenizer_path=SP_DIR, block_size=1, xxh3_seed=SEED, index_capacity=1 << 17)
    P = oracle.PrefixOracle(NAMES, 1, SEED)
    try:
        _set_view(_view(np.random.default_rng(1)), h, P)
        h.index_apply(5, stored=keys)
        P.record(NAMES[5], keys)
        h.index_apply(44, stored=keys[:40000])
        P.record(NAMES[44], keys[:40000])
        h.index_publish()
        P.upload()
        m = P.match(ids)
        assert m["hbm"][5] == 65536
        try:
            out = h.ingest_batch(batch.text, batch.offsets, 65536)
        except x.IngestError as e:
            code = e.code
        else:
            code = 0
            assert out["match"]["hbm"][0].tolist() == m["hbm"].tolist(), \
                "instance 5: device score %d, oracle %d" % (out["match"]["hbm"][0][5], m["hbm"][5])
        assert code == -1                                       # XLLM_ERR_INVALID_ARG
        # the same rule on the segmented entry point (it shares the batch core)
        seg = workload.SegmentBatch(np.zeros(0, np.uint8), np.zeros(1, np.int64), np.array([0, 1], np.int32),
                                    np.array([3], np.int32), np.arange(3, dtype=np.int32), np.zeros(1, bool),
                                    np.zeros(1, np.int32))
        with pytest.raises(x.IngestError) as ei:
            h.ingest_batch_segments(seg, 65536)
        assert ei.value.code == -1
        # 65 535 blocks: the row is truncated to 65 535 ids (status 1) and matched in full
        out = h.ingest_batch(batch.text, batch.offsets, 65535)
        assert out["status"][0] == 1 and out["n_ids"][0] == 65536
        assert (out["ids"][0] == ids[:65535]).all() and (out["keys"][0] == keys[:65535]).all()
        _check_match_route(P, ids[:65535], out["match"][0], out["routing"][0], "65535")
        assert out["match"]["hbm"][0][5] == 65535
        # keys only: 65 536 blocks hashed, no match
        out = h.ingest_batch(batch.text, batch.offsets, 65536, want_match=False)
        assert out["status"][0] == 0 and (out["keys"][0] == keys).all()
        # the host-pointer match refuses a 65 536-block request too
        with pytest.raises(x.IngestError) as ei:
            h.match_route(keys, np.zeros(1, np.int64), np.array([65536], np.int32))
        assert ei.value.code == -1
    finally:
        h.close()


# ----------------------------------------------------- D. the device-pointer entry points on a caller's stream
def test_device_pointer_path_on_a_caller_stream(oracle):
    """bench.py's device-resident step at a test size: encode_batch_device -> hash_blocks_device -> match_route_device
    back to back on a torch stream, no synchronisation in between.  All six outputs byte-identical to ingest_batch on
    the same batch, a sample equal to the oracle; then index_probe_device + score_route_device (the scoring half the
    sharded index uses) equal to index_get and to match_route_device."""
    import torch
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    n, T, bs = 4096, 1024, 128
    nb = T // bs
    rng = np.random.default_rng(4096)
    batch, meta = workload.make_prompts_exact_tokens(
        n, T, _word_counts(), seed=41, shared_prefix=dict(n_prefixes=16, frac=0.8, min_blocks=1, max_blocks=7,
                                                          block_tokens=bs))
    sp = oracle.SentencePieceOracle(SP_DIR)
    h = x.Ingest(tokenizer_path=SP_DIR, block_size=bs, xxh3_seed=SEED, index_capacity=1 << 16)
    P = oracle.PrefixOracle(NAMES, bs, SEED)
    try:
        _set_view(_view(rng), h, P)
        # index content: every shared prefix and a few whole prompts
        rows = [int(np.nonzero(meta["prefix_id"] == j)[0][0]) for j in range(16) if (meta["prefix_id"] == j).any()]
        rows += [int(r) for r in rng.integers(0, n, size=8)]
        key_rows = [oracle.block_hash_chain(sp.encode(batch.prompt(r)), bs, SEED) for r in rows]
        _apply(_events(key_rows, rng, per_window=80), h, P)
        ref = h.ingest_batch(batch.text, batch.offsets, T)
        assert (ref["status"] == 0).all() and (ref["n_ids"] == T).all()

        dev = torch.device("cuda", 0)
        stream = torch.cuda.Stream(device=dev)
        s = stream.cuda_stream
        d_text = torch.from_numpy(batch.text).to(dev)
        d_off = torch.from_numpy(batch.offsets).to(dev)
        d_ids = torch.full((n, T), -7, dtype=torch.int32, device=dev)
        d_nids = torch.full((n,), -7, dtype=torch.int32, device=dev)
        d_st = torch.full((n,), -7, dtype=torch.int32, device=dev)
        d_tok_start = torch.arange(n, device=dev, dtype=torch.int64) * T
        d_key_start = torch.arange(n, device=dev, dtype=torch.int64) * nb
        d_nblk = torch.full((n,), nb, dtype=torch.int32, device=dev)
        d_keys = torch.full((n, nb, 16), 0xEE, dtype=torch.uint8, device=dev)
        d_match = torch.full((n, 400), 0xAB, dtype=torch.uint8, device=dev)
        d_route = torch.full((n, 20), 0xCD, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        h.encode_batch_device(n, d_text.data_ptr(), d_off.data_ptr(), d_ids.data_ptr(), T, d_nids.data_ptr(),
                              d_st.data_ptr(), s)
        h.hash_blocks_device(n, d_ids.data_ptr(), d_tok_start.data_ptr(), d_nids.data_ptr(), d_keys.data_ptr(),
                             d_key_start.data_ptr(), s)
        h.match_route_device(n, d_keys.data_ptr(), n * nb, d_key_start.data_ptr(), d_nblk.data_ptr(),
                             d_match.data_ptr(), d_route.data_ptr(), s)
        stream.synchronize()
        assert d_ids.cpu().numpy().tobytes() == ref["ids"].tobytes()
        assert d_nids.cpu().numpy().tobytes() == ref["n_ids"].tobytes()
        assert d_st.cpu().numpy().tobytes() == ref["status"].tobytes()
        assert d_keys.cpu().numpy().tobytes() == ref["keys"].tobytes()
        assert d_match.cpu().numpy().tobytes() == ref["match"].tobytes()
        assert d_route.cpu().numpy().tobytes() == ref["routing"].tobytes()
        assert (ref["match"]["max_matched_block_num"] > 0).sum() > n // 4
        # a sample against the oracle
        sample = np.sort(rng.choice(n, size=64, replace=False))
        for r in sample:
            want = sp.encode(batch.prompt(int(r)))
            assert (ref["ids"][r] == want).all(), r
            _check_match_route(P, want, ref["match"][r], ref["routing"][r], int(r))

        # split probe / score: match_route_kernel<false> on one GPU
        d_masks = torch.full((n * nb, 3), -1, dtype=torch.int64, device=dev)
        d_m2 = torch.full((n, 400), 0x5A, dtype=torch.uint8, device=dev)
        d_r2 = torch.full((n, 20), 0x5A, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        h.index_probe_device(d_keys.data_ptr(), n * nb, d_masks.data_ptr(), s)
        h.score_route_device(n, d_masks.data_ptr(), d_key_start.data_ptr(), d_nblk.data_ptr(), d_m2.data_ptr(),
                             d_r2.data_ptr(), s)
        stream.synchronize()
        masks = d_masks.cpu().numpy().view(np.uint64)
        flat = ref["keys"].reshape(-1, 16)
        pref_rows = np.nonzero(meta["prefix_id"] >= 0)[0]
        picks = np.concatenate([pref_rows[:150] * nb, rng.integers(0, n * nb, size=250)])
        hits = 0
        for k in picks:
            found, mg = h.index_get(flat[k])
            assert masks[k].tolist() == mg, k
            assert P.get(flat[k]) == (found, mg), k
            hits += found
        assert 0 < hits < picks.size
        assert d_m2.cpu().numpy().tobytes() == ref["match"].tobytes()
        assert d_r2.cpu().numpy().tobytes() == ref["routing"].tobytes()

        # encode_batch_device: offsets that start inside the text (a row sub-range), strides that are not multiples
        # of 8 (1 021 truncates every row)
        r0, m = 100, 300
        for stride in (1021, 1030):
            e_ids = torch.full((m, stride), -7, dtype=torch.int32, device=dev)
            e_n = torch.full((m,), -7, dtype=torch.int32, device=dev)
            e_st = torch.full((m,), -7, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            h.encode_batch_device(m, d_text.data_ptr(), d_off[r0:].data_ptr(), e_ids.data_ptr(), stride,
                                  e_n.data_ptr(), e_st.data_ptr(), s)
            stream.synchronize()
            w_ids, w_n, w_st = h.encode_batch(batch.text, batch.offsets[r0:r0 + m + 1], stride)
            got_ids, got_n = e_ids.cpu().numpy(), e_n.cpu().numpy()
            assert (got_n == w_n).all() and (e_st.cpu().numpy() == w_st).all(), stride
            assert (w_st == (1 if stride < T else 0)).all()
            for r in range(m):
                have = min(int(w_n[r]), stride)
                assert (got_ids[r, :have] == w_ids[r, :have]).all(), (stride, r)
        # n_req = 0: returns at once, the (poisoned) outputs are left alone
        e_ids = torch.full((4, 16), -9, dtype=torch.int32, device=dev)
        e_n = torch.full((4,), -9, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        h.encode_batch_device(0, d_text.data_ptr(), d_off.data_ptr(), e_ids.data_ptr(), 16, e_n.data_ptr(),
                              e_n.data_ptr(), s)
        stream.synchronize()
        assert (e_ids.cpu() == -9).all() and (e_n.cpu() == -9).all()
    finally:
        h.close()


def test_device_encode_with_a_persistent_memo(oracle):
    """set_memo_policy(500) with batches of 200 requests: the device-pointer encode keeps its word memo across
    launches and clears it at the fourth one (its own age counter).  Every launch equals the oracle."""
    import torch
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    sp = oracle.SentencePieceOracle(SP_DIR)
    h = x.Ingest(tokenizer_path=SP_DIR)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    try:
        h.set_memo_policy(500)
        for k in range(6):
            texts = [t.encode() for t in workload.sentences(200, (1, 60), seed=300 + k)]
            if k == 3:
                texts[7] = "café 日本語 naïve".encode()
            b = workload.pack_prompts(texts)
            stride = 512
            d_text = torch.from_numpy(b.text).to(dev)
            d_off = torch.from_numpy(b.offsets).to(dev)
            d_ids = torch.zeros((b.n, stride), dtype=torch.int32, device=dev)
            d_n = torch.full((b.n,), -7, dtype=torch.int32, device=dev)
            d_st = torch.full((b.n,), -7, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            h.encode_batch_device(b.n, d_text.data_ptr(), d_off.data_ptr(), d_ids.data_ptr(), stride, d_n.data_ptr(),
                                  d_st.data_ptr(), stream.cuda_stream)
            stream.synchronize()
            w_ids, w_n = sp.encode_batch(b.text, b.offsets, stride)
            assert (w_n <= stride).all()
            assert (d_st.cpu().numpy() == 0).all(), k
            assert (d_n.cpu().numpy() == w_n).all(), k
            assert (d_ids.cpu().numpy() == w_ids).all(), k
    finally:
        h.close()


# ------------------------------------------------------------------- E. the bulk-copy hash variant
_BULK_CHILD = r"""
import json, os
import numpy as np
import torch
import xllm_service_b200 as x
from oracle import oracle as o

def csr(lengths):
    n_tok = np.asarray(lengths, dtype=np.int32)
    ts = np.zeros(len(lengths), dtype=np.int64)
    np.cumsum(n_tok[:-1], out=ts[1:])
    return ts, n_tok

res = {}
for seed in (1024, 0, 0xFFFFFFFF):
    rng = np.random.default_rng(1234 + seed % 97)
    h = x.Ingest(block_size=128, xxh3_seed=seed)
    lengths = [0, 1, 127, 128, 129, 255, 256, 257, 4096, 4095, 4097, 300, 8192, 128 * 37 + 5] + \
        list(rng.integers(0, 3000, size=150))
    ts, nt = csr(lengths)
    toks = rng.integers(-2**31, 2**31, size=int(nt.sum()), dtype=np.int64).astype(np.int32)
    keys, ks = h.hash_blocks(toks, ts, nt)
    want, want_off = o.block_hash_chain_batch(toks, np.concatenate([ts, [nt.sum()]]).astype(np.int64), 128, seed)
    res["ragged_%d" % seed] = bool(keys.shape == want.shape and (ks == want_off[:-1]).all() and (keys == want).all())
    h.close()

h = x.Ingest(block_size=128, xxh3_seed=1024)
rng = np.random.default_rng(99)
ts, nt = csr([257, 131, 1029, 515, 4099, 129] * 11)
toks = rng.integers(0, 152000, size=int(nt.sum())).astype(np.int32)
keys, _ = h.hash_blocks(toks, ts, nt)
want, _ = o.block_hash_chain_batch(toks, np.concatenate([ts, [nt.sum()]]), 128, 1024)
res["unaligned"] = bool((ts % 4 != 0).any() and (keys == want).all())

n, T = 8192, 4096
g = torch.Generator(device="cuda").manual_seed(5)
toks = torch.randint(0, 152000, (n, T), dtype=torch.int32, device="cuda", generator=g)
share = torch.arange(n, device="cuda") % 33
mask = (torch.arange(T, device="cuda")[None, :] // 128) < share[:, None]
toks = torch.where(mask, toks[0:1].expand(n, T), toks)
tok_start = torch.arange(n, device="cuda", dtype=torch.int64) * T
n_tok = torch.full((n,), T, dtype=torch.int32, device="cuda")
key_start = torch.arange(n, device="cuda", dtype=torch.int64) * (T // 128)
keys = torch.zeros((n, T // 128, 16), dtype=torch.uint8, device="cuda")
torch.cuda.synchronize()
h.hash_blocks_device(n, toks.data_ptr(), tok_start.data_ptr(), n_tok.data_ptr(), keys.data_ptr(), key_start.data_ptr())
torch.cuda.synchronize()
kc, tc, sh = keys.cpu().numpy(), toks.cpu().numpy(), share.cpu().numpy()
ok = all((kc[r] == o.block_hash_chain(tc[r], 128, 1024)).all() for r in (0, 1, 31, 32, 33, 1000, 4095, 8191))
same = (kc == kc[0:1]).all(axis=2)
res["full_size"] = bool(ok and (same == (np.arange(T // 128)[None, :] < sh[:, None]))[1:].all())
h.close()
print(json.dumps({"bulk": os.environ.get("XLLM_XXH3_BULK"), "cases": res}))
"""


def test_bulk_copy_hash_variant_in_a_child_process(oracle):
    """XLLM_XXH3_BULK=1 selects the cp.async.bulk + mbarrier staging of the 128-token hash kernel; it is read once per
    process, so a child process hashes the ragged, unaligned and full-size cases of test_gpu_xxh3.py with it."""
    env = dict(os.environ, XLLM_XXH3_BULK="1")
    p = subprocess.run([sys.executable, "-c", _BULK_CHILD], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    summary = json.loads(p.stdout.strip().splitlines()[-1])
    assert summary["bulk"] == "1"
    assert summary["cases"] == {"ragged_1024": True, "ragged_0": True, "ragged_4294967295": True, "unaligned": True,
                                "full_size": True}, summary
