"""ctypes loader for libxllm_ingest.so (built in-tree by `make lib` / __graft_entry__.build())."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# XLLM_INGEST_LIB: a diagnostics build of the same library (e.g. -DXLLM_EXP_STATS counters), developer use only
_LIB_PATH = os.environ.get("XLLM_INGEST_LIB") or os.path.join(_HERE, "libxllm_ingest.so")
_lib = None


class IngestError(RuntimeError):
    """A C-ABI entry point returned a negative XLLM_ERR_* code."""

    def __init__(self, code, msg):
        super().__init__(f"xllm_ingest error {code}: {msg}")
        self.code = code


def lib_path():
    return _LIB_PATH


class Config(ctypes.Structure):
    """xllm_ingest_config (include/xllm_ingest.h)."""
    _fields_ = [
        ("tokenizer_path", ctypes.c_char_p),
        ("block_size", ctypes.c_int32),
        ("xxh3_seed", ctypes.c_uint32),
        ("device", ctypes.c_int32),
        ("max_batch", ctypes.c_int32),
        ("max_batch_bytes", ctypes.c_int64),
        ("max_tokens", ctypes.c_int32),
        ("index_capacity", ctypes.c_int64),
        ("shard_world", ctypes.c_int32),
        ("shard_rank", ctypes.c_int32),
        ("nccl_unique_id", ctypes.c_void_p),
    ]


class ShardStats(ctypes.Structure):
    """xllm_shard_stats (include/xllm_ingest.h)."""
    _fields_ = [("bucket_ms", ctypes.c_float), ("exchange_out_ms", ctypes.c_float), ("probe_ms", ctypes.c_float),
                ("exchange_back_ms", ctypes.c_float), ("score_ms", ctypes.c_float),
                ("bucket_capacity", ctypes.c_int64), ("overflow_rounds", ctypes.c_int64)]


class TokenizerInfo(ctypes.Structure):
    """xllm_tokenizer_info (include/xllm_ingest.h)."""
    _fields_ = [(n, ctypes.c_int32) for n in ("n_pieces", "n_symbols", "n_pair_slots", "n_pairs", "split_mode",
                                              "max_unit_out", "byte_fallback", "unk_id", "trie_units",
                                              "avg_probe_x100", "max_probe")]


class MatchOut(ctypes.Structure):
    """xllm_match_out (include/xllm_ingest.h)."""
    _fields_ = [("max_block_num", ctypes.c_uint32), ("max_matched_block_num", ctypes.c_uint32),
                ("instances", ctypes.c_uint64), ("hbm_instance_score", ctypes.c_uint16 * 64),
                ("dram_instance_score", ctypes.c_uint16 * 64), ("ssd_instance_score", ctypes.c_uint16 * 64)]


class RoutingOut(ctypes.Structure):
    """xllm_routing_out (include/xllm_ingest.h)."""
    _fields_ = [("prefill_id", ctypes.c_int32), ("decode_id", ctypes.c_int32), ("ok", ctypes.c_int32),
                ("prefill_score", ctypes.c_float), ("decode_score", ctypes.c_float)]


MATCH_DTYPE = [("max_block_num", "<u4"), ("max_matched_block_num", "<u4"), ("instances", "<u8"),
               ("hbm", "<u2", (64,)), ("dram", "<u2", (64,)), ("ssd", "<u2", (64,))]
ROUTING_DTYPE = [("prefill_id", "<i4"), ("decode_id", "<i4"), ("ok", "<i4"), ("prefill_score", "<f4"),
                 ("decode_score", "<f4")]

class IngestIO(ctypes.Structure):
    """xllm_ingest_io (include/xllm_ingest.h)."""
    _fields_ = [("n_req", ctypes.c_int32), ("text", ctypes.c_void_p), ("offsets", ctypes.c_void_p),
                ("ids", ctypes.c_void_p), ("ids_stride", ctypes.c_int64), ("n_ids", ctypes.c_void_p),
                ("status", ctypes.c_void_p), ("keys", ctypes.c_void_p), ("keys_stride", ctypes.c_int64),
                ("match", ctypes.c_void_p), ("routing", ctypes.c_void_p), ("ids_u16", ctypes.c_void_p)]


class Segments(ctypes.Structure):
    """xllm_segments (include/xllm_ingest.h)."""
    _fields_ = [("n_segments", ctypes.c_int64), ("req_seg_start", ctypes.c_void_p), ("seg_len", ctypes.c_void_p),
                ("span_ids", ctypes.c_void_p), ("n_span_ids", ctypes.c_int64)]


_VP = ctypes.c_void_p
NFC_PROVE_INERT, NFC_VERIFY = 0, 1   # xllm_set_nfc_policy (include/xllm_ingest.h)


def _declare(L):
    L.xllm_last_error.restype = ctypes.c_char_p
    L.xllm_last_error.argtypes = []
    L.xllm_ingest_create.argtypes = [ctypes.POINTER(Config), ctypes.POINTER(_VP)]
    L.xllm_shard_unique_id.argtypes = [_VP]
    L.xllm_shard_owner.argtypes = [_VP, ctypes.c_int32]
    L.xllm_shard_last_stats.argtypes = [_VP, ctypes.POINTER(ShardStats)]
    L.xllm_ingest_clone.argtypes = [_VP, ctypes.POINTER(_VP)]
    L.xllm_ingest_destroy.argtypes = [_VP]
    L.xllm_ingest_destroy.restype = None
    L.xllm_hash_blocks.argtypes = [_VP, ctypes.c_int32, _VP, ctypes.c_int64, _VP, _VP, _VP, ctypes.c_int64, _VP]
    L.xllm_hash_blocks_device.argtypes = [_VP, ctypes.c_int32, _VP, _VP, _VP, _VP, _VP, _VP]
    L.xllm_xxh3_128bits_hash.argtypes = [_VP, _VP, _VP, ctypes.c_size_t, _VP]
    L.xllm_encode_batch.argtypes = [_VP, ctypes.c_int32, _VP, _VP, _VP, ctypes.c_int64, _VP, _VP]
    L.xllm_encode_batch_profile.argtypes = [_VP, ctypes.c_int32, _VP, _VP, ctypes.c_int64, _VP, _VP, _VP, ctypes.c_int32,
                                            ctypes.POINTER(ctypes.c_int32)]
    L.xllm_encode_batch_device.argtypes = [_VP, ctypes.c_int32, _VP, _VP, _VP, ctypes.c_int64, _VP, _VP, _VP]
    SZ = ctypes.c_size_t
    L.xllm_index_apply.argtypes = [_VP, ctypes.c_int32, _VP, SZ, _VP, SZ, _VP, SZ]
    L.xllm_index_put.argtypes = [_VP, _VP, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64]
    L.xllm_index_erase.argtypes = [_VP, _VP]
    L.xllm_index_publish.argtypes = [_VP]
    L.xllm_index_size.argtypes = [_VP, ctypes.POINTER(ctypes.c_int64)]
    L.xllm_index_clear_instance.argtypes = [_VP, ctypes.c_int32]
    L.xllm_index_stats.argtypes = [_VP] + [ctypes.POINTER(ctypes.c_int64)] * 3
    L.xllm_index_get.argtypes = [_VP, _VP, _VP, ctypes.POINTER(ctypes.c_int32)]
    L.xllm_set_instance.argtypes = [_VP, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32]
    L.xllm_set_load_metrics.argtypes = [_VP, ctypes.c_int32, ctypes.c_int32, ctypes.c_uint64, ctypes.c_float]
    L.xllm_match_route.argtypes = [_VP, ctypes.c_int32, _VP, ctypes.c_int64, _VP, _VP, _VP, _VP]
    L.xllm_match_route_device.argtypes = [_VP, ctypes.c_int32, _VP, ctypes.c_int64, _VP, _VP, _VP, _VP, _VP]
    L.xllm_index_probe_device.argtypes = [_VP, _VP, ctypes.c_int64, _VP, _VP]
    L.xllm_score_route_device.argtypes = [_VP, ctypes.c_int32, _VP, _VP, _VP, _VP, _VP, _VP]
    L.xllm_ingest_batch.argtypes = [_VP, ctypes.POINTER(IngestIO)]
    L.xllm_ingest_batch_segments.argtypes = [_VP, ctypes.POINTER(IngestIO), ctypes.POINTER(Segments)]
    L.xllm_index_put_bulk.argtypes = [_VP, ctypes.c_int64, _VP, _VP, _VP, _VP]
    L.xllm_index_export.argtypes = [_VP, ctypes.c_int64, _VP, _VP, _VP, _VP, ctypes.POINTER(ctypes.c_int64)]
    L.xllm_set_pipeline.argtypes = [_VP, ctypes.c_int32, ctypes.c_int64]
    L.xllm_set_memo_policy.argtypes = [_VP, ctypes.c_int64]
    L.xllm_set_nfc_policy.argtypes = [_VP, ctypes.c_int32]
    L.xllm_last_batch_stats.argtypes = [_VP, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]
    L.xllm_host_alloc.argtypes = [ctypes.POINTER(_VP), ctypes.c_size_t]
    L.xllm_host_free.argtypes = [_VP]
    L.xllm_host_free.restype = None
    L.xllm_tokenizer_probe.argtypes = [ctypes.c_char_p, ctypes.POINTER(TokenizerInfo)]
    L.xllm_vocab_size.argtypes = [_VP, ctypes.POINTER(ctypes.c_int32)]


def lib():
    """Load the CUDA library; raises (never falls back) when it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise IngestError(-3, f"{_LIB_PATH} not built: run `make lib` or __graft_entry__.build() "
                                  "(there is no CPU fallback)")
        L = ctypes.CDLL(_LIB_PATH)
        _declare(L)
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise IngestError(rc, lib().xllm_last_error().decode("utf-8", "replace"))


def tokenizer_probe(path):
    """Host-only parse of a tokenizer directory -> dict of table statistics (no GPU needed)."""
    info = TokenizerInfo()
    check(lib().xllm_tokenizer_probe(path.encode(), ctypes.byref(info)))
    return {n: getattr(info, n) for n, _ in TokenizerInfo._fields_}
