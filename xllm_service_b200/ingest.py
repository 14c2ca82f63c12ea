"""Host-side handle over the C-ABI (include/xllm_ingest.h)."""
import ctypes

import numpy as np

from . import _lib
from ._lib import Config, check


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None and a.size else None


class HostBuffer:
    """Page-locked host memory from xllm_host_alloc (placed on the GPU's NUMA node), viewed as a numpy array.
    Call with the device already selected (cudaSetDevice / torch.cuda.set_device)."""

    def __init__(self, shape, dtype):
        self._L = _lib.lib()
        self.array = None
        dt = np.dtype(dtype)
        n = int(np.prod(shape)) * dt.itemsize
        p = ctypes.c_void_p()
        check(self._L.xllm_host_alloc(ctypes.byref(p), n))
        self.ptr = p.value
        self.nbytes = n
        raw = (ctypes.c_uint8 * max(n, 1)).from_address(self.ptr)
        self.array = np.frombuffer(raw, dtype=dt, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if getattr(self, "ptr", None):
            self.array = None
            self._L.xllm_host_free(ctypes.c_void_p(self.ptr))
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Ingest:
    """One xllm_ingest_t handle.  Mirrors the hot-path knobs of the reference's Options
    (block_size, xxh3_128bits_seed, tokenizer_path: global_gflags.cpp:60,114-118)."""

    def __init__(self, tokenizer_path=None, block_size=128, xxh3_seed=1024, device=0, max_batch=0,
                 max_batch_bytes=0, max_tokens=0, index_capacity=0, shard_world=0, shard_rank=0,
                 nccl_unique_id=None):
        self._L = _lib.lib()
        self._h = ctypes.c_void_p()
        cfg = Config()
        cfg.tokenizer_path = tokenizer_path.encode() if tokenizer_path else None
        cfg.block_size = block_size
        cfg.xxh3_seed = xxh3_seed
        cfg.device = device
        cfg.max_batch = max_batch
        cfg.max_batch_bytes = max_batch_bytes
        cfg.max_tokens = max_tokens
        cfg.index_capacity = index_capacity
        # hash-range-sharded index: collective create (every rank, same 128-byte id: sharded.create_sharded)
        cfg.shard_world = shard_world
        cfg.shard_rank = shard_rank
        self._uid = ctypes.create_string_buffer(bytes(nccl_unique_id), 128) if nccl_unique_id is not None else None
        cfg.nccl_unique_id = ctypes.cast(self._uid, ctypes.c_void_p) if self._uid is not None else None
        self.block_size = block_size or 128
        self.seed = xxh3_seed
        check(self._L.xllm_ingest_create(ctypes.byref(cfg), ctypes.byref(self._h)))

    def close(self):
        if self._h:
            self._L.xllm_ingest_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ hash
    def xxh3_128bits_hash(self, prev, token_ids) -> bytes:
        """Drop-in for xxh3_128bits_hash(pre_hash_value, token_ids, hash_value)
        (xllm_service/common/hash_util.h:56-58)."""
        t = np.ascontiguousarray(token_ids, dtype=np.int32)
        out = ctypes.create_string_buffer(16)
        pbuf = ctypes.create_string_buffer(bytes(prev), 16) if prev is not None else None
        check(self._L.xllm_xxh3_128bits_hash(self._h, pbuf, _ptr(t), t.size, out))
        return out.raw

    def hash_blocks(self, tokens, tok_start, n_tok, key_start=None):
        """Host-buffer batch chain (global_kvcache_mgr.cpp:76-94).  Returns (keys uint8[n_keys,16], key_start)."""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        tok_start = np.ascontiguousarray(tok_start, dtype=np.int64)
        n_tok = np.ascontiguousarray(n_tok, dtype=np.int32)
        n = n_tok.size
        nb = n_tok.astype(np.int64) // self.block_size
        if key_start is None:
            key_start = np.zeros(n, dtype=np.int64)
            if n:
                np.cumsum(nb[:-1], out=key_start[1:])
        key_start = np.ascontiguousarray(key_start, dtype=np.int64)
        n_keys = int((key_start + nb).max()) if n else 0
        keys = np.zeros((n_keys, 16), dtype=np.uint8)
        check(self._L.xllm_hash_blocks(self._h, n, _ptr(tokens), tokens.size, _ptr(tok_start), _ptr(n_tok),
                                       _ptr(keys), n_keys, _ptr(key_start)))
        return keys, key_start

    def hash_blocks_device(self, n_req, d_tokens, d_tok_start, d_n_tok, d_keys, d_key_start, stream=None):
        """Device-pointer batch chain; arguments are integer device addresses (e.g. torch .data_ptr())."""
        check(self._L.xllm_hash_blocks_device(self._h, n_req, d_tokens, d_tok_start, d_n_tok, d_keys, d_key_start,
                                              stream))

    # -------------------------------------------------------------- tokenize
    def vocab_size(self):
        out = ctypes.c_int32()
        check(self._L.xllm_vocab_size(self._h, ctypes.byref(out)))
        return out.value

    def encode_batch(self, text, offsets, ids_stride):
        """Batch Tokenizer::encode over host buffers.  text: uint8 array, offsets int64[n+1].
        Returns (ids int32[n, ids_stride], n_ids int32[n], status int32[n])."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n = offsets.size - 1
        ids = np.zeros((n, ids_stride), dtype=np.int32)
        n_ids = np.zeros(n, dtype=np.int32)
        status = np.zeros(n, dtype=np.int32)
        check(self._L.xllm_encode_batch(self._h, n, _ptr(text), _ptr(offsets), _ptr(ids), ids_stride, _ptr(n_ids),
                                        _ptr(status)))
        return ids, n_ids, status

    def encode_batch_profile(self, text, offsets, ids_stride):
        """xllm_encode_batch_profile -> (n_ids, status, warp_ns uint64[n_warps]): per-warp busy time of the tokenizer's
        persistent grid for this batch."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n = offsets.size - 1
        n_ids, status = np.zeros(n, np.int32), np.zeros(n, np.int32)
        cap = 1 << 16
        warp = np.zeros(cap, np.uint64)
        nw = ctypes.c_int32()
        check(self._L.xllm_encode_batch_profile(self._h, n, _ptr(text), _ptr(offsets), ids_stride, _ptr(n_ids),
                                                _ptr(status), _ptr(warp), cap, ctypes.byref(nw)))
        return n_ids, status, warp[:min(nw.value, cap)].copy()

    def encode(self, text: bytes):
        """Single-request Tokenizer::encode (tokenizer.h:32-33): returns the id list; raises on failure
        (the reference returns false, scheduler.cpp:129-132)."""
        if isinstance(text, str):
            text = text.encode("utf-8")
        t = np.frombuffer(text, dtype=np.uint8)
        off = np.array([0, t.size], dtype=np.int64)
        stride = max(16, 3 * t.size + 8)
        ids, n_ids, status = self.encode_batch(t, off, stride)
        if status[0] == 1:  # XLLM_ENC_TRUNCATED: n_ids holds the needed size
            ids, n_ids, status = self.encode_batch(t, off, int(n_ids[0]))
        if status[0] < 0:
            raise _lib.IngestError(int(status[0]), "encode failed")
        return ids[0, :n_ids[0]].tolist()

    def encode_batch_device(self, n_req, d_text, d_offsets, d_ids, ids_stride, d_n_ids, d_status, stream=None):
        check(self._L.xllm_encode_batch_device(self._h, n_req, d_text, d_offsets, d_ids, ids_stride, d_n_ids,
                                               d_status, stream))

    # ---------------------------------------------------------- prefix index
    @staticmethod
    def _keys(keys):
        if keys is None:
            return np.zeros((0, 16), np.uint8)
        return np.ascontiguousarray(np.asarray(keys, dtype=np.uint8).reshape(-1, 16))

    def index_put_bulk(self, keys, hbm, dram, ssd):
        """Bulk replica PUT (update_kvcache / start-up load, global_kvcache_mgr.cpp:47-51,133-175); staged."""
        k = self._keys(keys)
        m = [np.ascontiguousarray(x, dtype=np.uint64) for x in (hbm, dram, ssd)]
        assert all(x.size == k.shape[0] for x in m)
        check(self._L.xllm_index_put_bulk(self._h, k.shape[0], _ptr(k), _ptr(m[0]), _ptr(m[1]), _ptr(m[2])))

    def index_export(self):
        """Snapshot of the published index: (keys uint8[n,16], hbm, dram, ssd uint64[n]), order unspecified."""
        n = ctypes.c_int64()
        cap = max(1, self.index_size())
        while True:
            keys = np.zeros((cap, 16), np.uint8)
            m = [np.zeros(cap, np.uint64) for _ in range(3)]
            rc = self._L.xllm_index_export(self._h, cap, _ptr(keys), _ptr(m[0]), _ptr(m[1]), _ptr(m[2]), ctypes.byref(n))
            if rc == -6 and n.value > cap:      # grew in between: retry with the reported size
                cap = n.value
                continue
            check(rc)
            return keys[:n.value], m[0][:n.value], m[1][:n.value], m[2][:n.value]

    def index_apply(self, instance_id, stored=None, offload=None, removed=None):
        """GlobalKVCacheMgr::record_updated_kvcaches (global_kvcache_mgr.cpp:177-225); staged."""
        s, o, r = self._keys(stored), self._keys(offload), self._keys(removed)
        check(self._L.xllm_index_apply(self._h, instance_id, _ptr(s), s.shape[0], _ptr(o), o.shape[0], _ptr(r),
                                       r.shape[0]))

    def index_put(self, key, hbm_mask=0, dram_mask=0, ssd_mask=0):
        k = self._keys(key)
        check(self._L.xllm_index_put(self._h, _ptr(k), hbm_mask, dram_mask, ssd_mask))

    def index_erase(self, key):
        k = self._keys(key)
        check(self._L.xllm_index_erase(self._h, _ptr(k)))

    def index_publish(self):
        """upload_kvcache (global_kvcache_mgr.cpp:227-247): staged events become visible to match."""
        check(self._L.xllm_index_publish(self._h))

    def shard_last_stats(self):
        """Device milliseconds of the last sharded match round + message capacity + overflow repeats."""
        st = _lib.ShardStats()
        check(self._L.xllm_shard_last_stats(self._h, ctypes.byref(st)))
        return {n: getattr(st, n) for n, _ in _lib.ShardStats._fields_}

    def index_clear_instance(self, instance_id):
        """Drop one instance from every entry of the published index (entries left empty are erased)."""
        check(self._L.xllm_index_clear_instance(self._h, instance_id))

    def index_stats(self):
        """(live keys, tombstones, in-place rebuilds) as of the last publish."""
        v = [ctypes.c_int64() for _ in range(3)]
        check(self._L.xllm_index_stats(self._h, *[ctypes.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def index_size(self):
        n = ctypes.c_int64()
        check(self._L.xllm_index_size(self._h, ctypes.byref(n)))
        return n.value

    def index_get(self, key):
        k = self._keys(key)
        m = np.zeros(3, dtype=np.uint64)
        f = ctypes.c_int32()
        check(self._L.xllm_index_get(self._h, _ptr(k), _ptr(m), ctypes.byref(f)))
        return bool(f.value), [int(x) for x in m]

    def set_instance(self, instance_id, type_, schedulable=True):
        check(self._L.xllm_set_instance(self._h, instance_id, type_, int(schedulable)))

    def set_load_metrics(self, instance_id, waiting, usage, has_metrics=True):
        check(self._L.xllm_set_load_metrics(self._h, instance_id, int(has_metrics), int(waiting), float(usage)))

    def match_route(self, keys, key_start, n_blocks):
        """GlobalKVCacheMgr::match + CacheAwareRouting::select_instances_pair over host buffers.
        Returns (match structured array, routing structured array)."""
        keys = self._keys(keys)
        key_start = np.ascontiguousarray(key_start, dtype=np.int64)
        n_blocks = np.ascontiguousarray(n_blocks, dtype=np.int32)
        n = n_blocks.size
        match = np.zeros(n, dtype=_lib.MATCH_DTYPE)
        routing = np.zeros(n, dtype=_lib.ROUTING_DTYPE)
        assert match.itemsize == 400 and routing.itemsize == 20
        check(self._L.xllm_match_route(self._h, n, _ptr(keys), keys.shape[0], _ptr(key_start), _ptr(n_blocks),
                                       _ptr(match), _ptr(routing)))
        return match, routing

    def match_route_device(self, n_req, d_keys, n_keys, d_key_start, d_n_blocks, d_match, d_routing, stream=None):
        check(self._L.xllm_match_route_device(self._h, n_req, d_keys, n_keys, d_key_start, d_n_blocks, d_match,
                                              d_routing, stream))

    def index_probe_device(self, d_keys, n_keys, d_masks3, stream=None):
        check(self._L.xllm_index_probe_device(self._h, d_keys, n_keys, d_masks3, stream))

    def score_route_device(self, n_req, d_masks3, d_key_start, d_n_blocks, d_match, d_routing, stream=None):
        check(self._L.xllm_score_route_device(self._h, n_req, d_masks3, d_key_start, d_n_blocks, d_match, d_routing,
                                              stream))

    # ------------------------------------------------------- the whole path
    def set_pipeline(self, chunk_requests, chunk_bytes):
        check(self._L.xllm_set_pipeline(self._h, chunk_requests, chunk_bytes))

    def set_memo_policy(self, persist_requests):
        """0: every encode launch clears its word memo (default); N > 0: a memo is kept until it has seen N requests."""
        check(self._L.xllm_set_memo_policy(self._h, persist_requests))

    def set_nfc_policy(self, policy):
        """Tokenizers with `normalizer: NFC`: 0 (XLLM_NFC_PROVE_INERT, default) accepts a request only when every char
        is NFC-inert; 1 (XLLM_NFC_VERIFY) checks exactly whether it is in NFC.  Refused requests get status -5."""
        check(self._L.xllm_set_nfc_policy(self._h, policy))

    def last_batch_stats(self):
        """(chunks, kernel launches) of the most recent ingest_batch on this handle."""
        c, k = ctypes.c_int32(), ctypes.c_int32()
        check(self._L.xllm_last_batch_stats(self._h, ctypes.byref(c), ctypes.byref(k)))
        return c.value, k.value

    def ingest_batch_ptrs(self, n_req, text, offsets, ids, ids_stride, n_ids, status, keys=0, keys_stride=0,
                          match=0, routing=0, ids_u16=0):
        """xllm_ingest_batch over raw host addresses (ints), e.g. pinned torch tensors' data_ptr().  ids_u16: address
        of a uint16 [n_req, ids_stride] buffer for the narrow download (then `ids` may be 0)."""
        io = _lib.IngestIO(n_req, text, offsets, ids or None, ids_stride, n_ids, status, keys or None, keys_stride,
                           match or None, routing or None, ids_u16 or None)
        check(self._L.xllm_ingest_batch(self._h, ctypes.byref(io)))

    def ingest_batch(self, text, offsets, ids_stride, want_keys=True, want_match=True, ids_u16=False):
        """tokenize + block-hash + match + route for a batch of prompts (numpy host buffers).
        Returns dict(ids, n_ids, status, keys, match, routing); ids_u16=True takes the narrow download (ids is then a
        uint16 array)."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n = offsets.size - 1
        ks = ids_stride // self.block_size
        out = {"ids": np.zeros((n, ids_stride), np.uint16 if ids_u16 else np.int32), "n_ids": np.zeros(n, np.int32),
               "status": np.zeros(n, np.int32), "keys": None, "match": None, "routing": None}
        if want_keys:
            out["keys"] = np.zeros((n, ks, 16), np.uint8)
        if want_match:
            out["match"] = np.zeros(n, dtype=_lib.MATCH_DTYPE)
            out["routing"] = np.zeros(n, dtype=_lib.ROUTING_DTYPE)
        a = lambda x: x.ctypes.data if x is not None and x.size else 0  # noqa: E731
        self.ingest_batch_ptrs(n, a(text), a(offsets), 0 if ids_u16 else a(out["ids"]), ids_stride, a(out["n_ids"]),
                               a(out["status"]), a(out["keys"]), ks if want_keys else 0, a(out["match"]),
                               a(out["routing"]), a(out["ids"]) if ids_u16 else 0)
        return out

    def ingest_batch_segments_ptrs(self, n_req, text, offsets, ids, ids_stride, n_ids, status, n_segments,
                                   req_seg_start, seg_len, span_ids, n_span_ids, keys=0, keys_stride=0, match=0,
                                   routing=0):
        """xllm_ingest_batch_segments over raw host addresses (ints)."""
        io = _lib.IngestIO(n_req, text, offsets, ids, ids_stride, n_ids, status, keys or None, keys_stride,
                           match or None, routing or None)
        sg = _lib.Segments(n_segments, req_seg_start, seg_len, span_ids or None, n_span_ids)
        check(self._L.xllm_ingest_batch_segments(self._h, ctypes.byref(io), ctypes.byref(sg)))

    def ingest_batch_segments(self, seg_batch, ids_stride, want_keys=True, want_match=True):
        """Requests made of text pieces and ready-made id spans (workload.SegmentBatch) -> the same dict as
        ingest_batch.  Text pieces are tokenised like independent Tokenizer::encode calls and appended; id spans are
        copied; keys / match / routing run over the concatenation."""
        b = seg_batch
        text = np.ascontiguousarray(b.text, dtype=np.uint8)
        offsets = np.ascontiguousarray(b.offsets, dtype=np.int64)
        rss = np.ascontiguousarray(b.req_seg_start, dtype=np.int32)
        sl = np.ascontiguousarray(b.seg_len, dtype=np.int32)
        span = np.ascontiguousarray(b.span_ids, dtype=np.int32)
        n = rss.size - 1
        ks = ids_stride // self.block_size
        out = {"ids": np.zeros((n, ids_stride), np.int32), "n_ids": np.zeros(n, np.int32),
               "status": np.zeros(n, np.int32), "keys": None, "match": None, "routing": None}
        if want_keys:
            out["keys"] = np.zeros((n, ks, 16), np.uint8)
        if want_match:
            out["match"] = np.zeros(n, dtype=_lib.MATCH_DTYPE)
            out["routing"] = np.zeros(n, dtype=_lib.ROUTING_DTYPE)
        a = lambda x: x.ctypes.data if x is not None and x.size else 0  # noqa: E731
        self.ingest_batch_segments_ptrs(n, a(text), offsets.ctypes.data, a(out["ids"]), ids_stride, a(out["n_ids"]),
                                        a(out["status"]), sl.size, rss.ctypes.data, a(sl), a(span), span.size,
                                        a(out["keys"]), ks if want_keys else 0, a(out["match"]), a(out["routing"]))
        return out
