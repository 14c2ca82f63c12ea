"""ctypes bindings of oracle/liboracle.so (the C/C++ restatement of the reference's
CPU hot path).  TEST INFRASTRUCTURE ONLY — see oracle/__init__.py."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")
_lib = None

c_u8p = ctypes.POINTER(ctypes.c_uint8)
c_i32p = ctypes.POINTER(ctypes.c_int32)
c_i64p = ctypes.POINTER(ctypes.c_int64)


def build():
    """(Re)build liboracle.so with make; a no-op when it is up to date."""
    subprocess.check_call(["make", "-s", "oracle"], cwd=os.path.dirname(_HERE))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = ctypes.CDLL(_LIB_PATH)
        L.oracle_xxh3_128_with_seed.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_void_p]
        L.oracle_xxh3_128_with_seed.restype = None
        L.oracle_xxh3_128bits_hash.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32,
                                               ctypes.c_void_p]
        L.oracle_xxh3_128bits_hash.restype = ctypes.c_int
        L.oracle_block_hash_chain.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_uint32,
                                              ctypes.c_void_p]
        L.oracle_block_hash_chain.restype = ctypes.c_long
        L.oracle_block_hash_chain_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                                    ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p,
                                                    ctypes.c_void_p]
        L.oracle_block_hash_chain_batch.restype = ctypes.c_long
        L.oracle_sp_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        L.oracle_sp_load.restype = ctypes.c_void_p
        L.oracle_sp_free.argtypes = [ctypes.c_void_p]
        L.oracle_sp_free.restype = None
        L.oracle_sp_piece_count.argtypes = [ctypes.c_void_p]
        L.oracle_sp_normalize.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p,
                                          ctypes.c_size_t]
        L.oracle_sp_normalize.restype = ctypes.c_long
        L.oracle_sp_encode.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p,
                                       ctypes.c_size_t]
        L.oracle_sp_encode.restype = ctypes.c_long
        L.oracle_sp_encode_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                             ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int]
        VP = ctypes.c_void_p
        L.oracle_index_new.restype = VP
        L.oracle_index_free.argtypes = [VP]
        L.oracle_index_free.restype = None
        L.oracle_index_size.argtypes = [VP]
        L.oracle_index_size.restype = ctypes.c_long
        L.oracle_index_record.argtypes = [VP, ctypes.c_char_p, VP, ctypes.c_size_t, VP, ctypes.c_size_t, VP,
                                          ctypes.c_size_t]
        L.oracle_index_record.restype = None
        L.oracle_index_upload.argtypes = [VP]
        L.oracle_index_upload.restype = None
        L.oracle_index_put.argtypes = [VP, VP, VP, ctypes.c_int, VP, ctypes.c_int, VP, ctypes.c_int]
        L.oracle_index_put.restype = None
        L.oracle_index_delete.argtypes = [VP, VP]
        L.oracle_index_delete.restype = None
        L.oracle_index_get.argtypes = [VP, VP, VP, ctypes.c_int, VP]
        L.oracle_index_match.argtypes = [VP, VP, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_uint32, VP, ctypes.c_int,
                                         VP, VP, VP, VP]
        L.oracle_index_match.restype = None
        L.oracle_registry_new.restype = VP
        L.oracle_registry_free.argtypes = [VP]
        L.oracle_registry_free.restype = None
        L.oracle_registry_set_instance.argtypes = [VP, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
        L.oracle_registry_set_instance.restype = None
        L.oracle_registry_set_load.argtypes = [VP, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_float]
        L.oracle_registry_set_load.restype = None
        L.oracle_registry_clear_load.argtypes = [VP, ctypes.c_char_p]
        L.oracle_registry_clear_load.restype = None
        L.oracle_route_car.argtypes = [VP, VP, VP, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_uint32, VP, ctypes.c_int,
                                       VP, VP, VP, VP, VP, VP]
        L.oracle_tik_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        L.oracle_tik_load.restype = VP
        L.oracle_tik_free.argtypes = [VP]
        L.oracle_tik_free.restype = None
        L.oracle_tik_vocab_size.argtypes = [VP]
        L.oracle_tik_vocab_size.restype = ctypes.c_long
        L.oracle_tik_encode.argtypes = [VP, ctypes.c_char_p, ctypes.c_size_t, VP, ctypes.c_size_t]
        L.oracle_tik_encode.restype = ctypes.c_long
        L.oracle_hf_new.argtypes = [VP, VP, ctypes.c_size_t, ctypes.c_char_p, VP, VP, VP, ctypes.c_size_t]
        L.oracle_hf_new.restype = VP
        L.oracle_hf_configure.argtypes = [VP, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, VP, VP,
                                          ctypes.c_size_t]
        L.oracle_hf_configure.restype = None
        L.oracle_hf_free.argtypes = [VP]
        L.oracle_hf_free.restype = None
        L.oracle_hf_encode.argtypes = [VP, ctypes.c_char_p, ctypes.c_size_t, VP, ctypes.c_size_t]
        L.oracle_hf_encode.restype = ctypes.c_long
        L.oracle_ingest_batch.argtypes = [VP, VP, VP, VP, VP, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_uint32, VP,
                                          ctypes.c_int, ctypes.c_int, VP, ctypes.c_int64, VP, VP, VP, VP]
        _lib = L
    return _lib


def xxh3_128_with_seed(data: bytes, seed: int) -> bytes:
    """XXH3_128bits_withSeed; returns the XXH128_hash_t struct bytes (low64 LE || high64 LE)."""
    out = ctypes.create_string_buffer(16)
    buf = ctypes.create_string_buffer(bytes(data), len(data)) if len(data) else None
    lib().oracle_xxh3_128_with_seed(buf, len(data), seed, out)
    return out.raw


def xxh3_128bits_hash(prev, token_ids, seed=1024) -> bytes:
    """hash_util.cpp:18-45.  prev: 16 bytes or None."""
    t = np.ascontiguousarray(token_ids, dtype=np.int32)
    out = ctypes.create_string_buffer(16)
    pbuf = ctypes.create_string_buffer(bytes(prev), 16) if prev is not None else None
    rc = lib().oracle_xxh3_128bits_hash(pbuf, t.ctypes.data, t.size, seed, out)
    if rc != 0:
        raise ValueError("key size is too small (hash_util.cpp:33)")
    return out.raw


def block_hash_chain(token_ids, block_size=128, seed=1024) -> np.ndarray:
    """Chain of global_kvcache_mgr.cpp:76-94 -> uint8 [n_blocks, 16]."""
    t = np.ascontiguousarray(token_ids, dtype=np.int32)
    nb = t.size // block_size
    keys = np.zeros((nb, 16), dtype=np.uint8)
    rc = lib().oracle_block_hash_chain(t.ctypes.data, t.size, block_size, seed, keys.ctypes.data)
    if rc < 0:
        raise ValueError("oracle_block_hash_chain failed")
    return keys


def block_hash_chain_batch(tokens, tok_offsets, block_size=128, seed=1024):
    """CSR batch: tokens int32[total], tok_offsets int64[n+1] -> (keys uint8[total_blocks,16], key_offsets int64[n+1])."""
    tokens = np.ascontiguousarray(tokens, dtype=np.int32)
    tok_offsets = np.ascontiguousarray(tok_offsets, dtype=np.int64)
    n = tok_offsets.size - 1
    nb = (tok_offsets[1:] - tok_offsets[:-1]) // block_size
    key_offsets = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(nb, out=key_offsets[1:])
    keys = np.zeros((int(key_offsets[-1]), 16), dtype=np.uint8)
    rc = lib().oracle_block_hash_chain_batch(tokens.ctypes.data, tok_offsets.ctypes.data, n, block_size, seed,
                                             keys.ctypes.data, key_offsets.ctypes.data)
    if rc < 0:
        raise ValueError("oracle_block_hash_chain_batch failed")
    return keys, key_offsets


class SentencePieceOracle:
    """SentencePieceTokenizer (xllm_service/tokenizer/sentencepiece_tokenizer.cpp:47-168) over the
    C++ restatement of libsentencepiece's BPE path (oracle/sp_oracle.cc)."""

    def __init__(self, model_dir_or_file):
        path = model_dir_or_file
        if os.path.isdir(path):
            path = os.path.join(path, "tokenizer.model")  # tokenizer_args.h:37 default vocab_file
        err = ctypes.create_string_buffer(512)
        self._h = lib().oracle_sp_load(path.encode(), err, 512)
        if not self._h:
            raise ValueError("oracle_sp_load: " + err.value.decode())

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().oracle_sp_free(self._h)
                self._h = None
        except Exception:  # interpreter shutdown
            pass

    def vocab_size(self):
        return lib().oracle_sp_piece_count(self._h)

    def normalize(self, text: bytes) -> bytes:
        cap = 3 * len(text) + 16
        out = ctypes.create_string_buffer(cap)
        n = lib().oracle_sp_normalize(self._h, text, len(text), out, cap)
        if n > cap:  # a charsmap replacement longer than 3x its key (e.g. U+FDFA)
            cap = n
            out = ctypes.create_string_buffer(cap)
            n = lib().oracle_sp_normalize(self._h, text, len(text), out, cap)
        return out.raw[:n]

    def encode(self, text: bytes):
        cap = len(text) * 3 + 16  # every byte can become a byte-fallback id; dummy prefix adds one
        out = np.zeros(cap, dtype=np.int32)
        n = lib().oracle_sp_encode(self._h, text, len(text), out.ctypes.data, cap)
        if n > cap:  # charsmap expansions (e.g. U+FDFA -> 18 chars)
            cap = n
            out = np.zeros(cap, dtype=np.int32)
            n = lib().oracle_sp_encode(self._h, text, len(text), out.ctypes.data, cap)
        return out[:n].copy()

    def encode_batch(self, text_u8, offsets, ids_stride, n_threads=1):
        """CSR batch -> (ids int32[n, ids_stride] zero padded, n_ids int32[n])."""
        text_u8 = np.ascontiguousarray(text_u8, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n = offsets.size - 1
        ids = np.zeros((n, ids_stride), dtype=np.int32)
        n_ids = np.zeros(n, dtype=np.int32)
        lib().oracle_sp_encode_batch(self._h, text_u8.ctypes.data, offsets.ctypes.data, n, ids.ctypes.data,
                                     ids_stride, n_ids.ctypes.data, n_threads)
        return ids, n_ids


def _name_array(names):
    arr = (ctypes.c_char_p * len(names))(*[n.encode() for n in names])
    return arr


def _keys_buf(keys):
    """list of 16-byte keys / uint8 [n,16] -> (contiguous uint8 array, n)."""
    a = np.ascontiguousarray(np.asarray(keys, dtype=np.uint8).reshape(-1, 16)) if len(keys) else np.zeros((0, 16),
                                                                                                         np.uint8)
    return a, a.shape[0]


class PrefixOracle:
    """GlobalKVCacheMgr + InstanceMgr::get_load_metrics + CacheAwareRouting with the reference's own
    containers (oracle/prefix_oracle.cc).  Instances are NAMES here, exactly as in the reference;
    `names` (id -> name) only translates results to the id space the device path uses."""
    DEFAULT, PREFILL, DECODE, MIX = 0, 1, 2, 3

    def __init__(self, names, block_size=128, seed=1024):
        self.names = list(names)
        self._names = _name_array(self.names)
        self.block_size, self.seed = block_size, seed
        self._ix = lib().oracle_index_new()
        self._reg = lib().oracle_registry_new()

    def __del__(self):
        try:
            lib().oracle_index_free(self._ix)
            lib().oracle_registry_free(self._reg)
        except Exception:
            pass

    # write side
    def record(self, name, stored=(), offload=(), removed=()):
        s, ns = _keys_buf(stored)
        o, no = _keys_buf(offload)
        r, nr = _keys_buf(removed)
        lib().oracle_index_record(self._ix, name.encode(), s.ctypes.data, ns, o.ctypes.data, no, r.ctypes.data, nr)

    def upload(self):
        lib().oracle_index_upload(self._ix)

    def put(self, key, hbm=(), dram=(), ssd=()):
        k = np.ascontiguousarray(np.frombuffer(bytes(key), dtype=np.uint8))
        lib().oracle_index_put(self._ix, k.ctypes.data, _name_array(list(hbm)), len(hbm), _name_array(list(dram)),
                               len(dram), _name_array(list(ssd)), len(ssd))

    def delete(self, key):
        k = np.ascontiguousarray(np.frombuffer(bytes(key), dtype=np.uint8))
        lib().oracle_index_delete(self._ix, k.ctypes.data)

    def size(self):
        return lib().oracle_index_size(self._ix)

    def get(self, key):
        k = np.ascontiguousarray(np.frombuffer(bytes(key), dtype=np.uint8))
        m = np.zeros(3, dtype=np.uint64)
        found = lib().oracle_index_get(self._ix, k.ctypes.data, self._names, len(self.names), m.ctypes.data)
        return bool(found), [int(x) for x in m]

    # registry
    def set_instance(self, name, type_, schedulable=True):
        lib().oracle_registry_set_instance(self._reg, name.encode(), type_, int(schedulable))

    def set_load(self, name, waiting, usage):
        lib().oracle_registry_set_load(self._reg, name.encode(), int(waiting), float(usage))

    def clear_load(self, name):
        lib().oracle_registry_clear_load(self._reg, name.encode())

    # read side
    def match(self, tokens):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        n = len(self.names)
        scores = np.zeros((3, n), dtype=np.uint32)
        inst = ctypes.c_uint64()
        mb, mm = ctypes.c_uint32(), ctypes.c_uint32()
        lib().oracle_index_match(self._ix, t.ctypes.data, t.size, self.block_size, self.seed, self._names, n,
                                 scores.ctypes.data, ctypes.byref(inst), ctypes.byref(mb), ctypes.byref(mm))
        return {"hbm": scores[0], "dram": scores[1], "ssd": scores[2], "instances": inst.value,
                "max_block_num": mb.value, "max_matched_block_num": mm.value}

    def route(self, tokens):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        pid, did = ctypes.c_int(), ctypes.c_int()
        pb, db = ctypes.c_float(), ctypes.c_float()
        pa, da = ctypes.c_uint64(), ctypes.c_uint64()
        ok = lib().oracle_route_car(self._ix, self._reg, t.ctypes.data, t.size, self.block_size, self.seed,
                                    self._names, len(self.names), ctypes.byref(pid), ctypes.byref(did),
                                    ctypes.byref(pb), ctypes.byref(db), ctypes.byref(pa), ctypes.byref(da))
        return {"ok": bool(ok), "prefill_id": pid.value, "decode_id": did.value, "prefill_score": pb.value,
                "decode_score": db.value, "prefill_argmax": pa.value, "decode_argmax": da.value}


def ingest_batch(sp, prefix, text_u8, offsets, ids_stride, n_threads=1, want_ids=True):
    """Scheduler::schedule's encode + select_instances_pair for every request of a CSR batch, one request
    at a time per worker thread.  sp: SentencePieceOracle; prefix: PrefixOracle or None.
    Returns dict(ids, n_ids, prefill_id, decode_id, ok)."""
    text_u8 = np.ascontiguousarray(text_u8, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    n = offsets.size - 1
    ids = np.zeros((n, ids_stride), dtype=np.int32) if want_ids else None
    n_ids = np.zeros(n, np.int32)
    pid = np.full(n, -1, np.int32)
    did = np.full(n, -1, np.int32)
    ok = np.zeros(n, np.int32)
    lib().oracle_ingest_batch(sp._h, prefix._ix if prefix else None, prefix._reg if prefix else None,
                              text_u8.ctypes.data, offsets.ctypes.data, n,
                              prefix.block_size if prefix else 128, prefix.seed if prefix else 1024,
                              prefix._names if prefix else None, len(prefix.names) if prefix else 0, n_threads,
                              ids.ctypes.data if want_ids else None, ids_stride, n_ids.ctypes.data, pid.ctypes.data,
                              did.ctypes.data, ok.ctypes.data)
    return {"ids": ids, "n_ids": n_ids, "prefill_id": pid, "decode_id": did, "ok": ok}


class TiktokenOracle:
    """TiktokenTokenizer as the service configures it (no regex pattern: the whole text is one piece);
    oracle/tiktoken_oracle.cc restating tiktoken_tokenizer.cpp:115-294."""

    def __init__(self, model_dir_or_file):
        path = model_dir_or_file
        if os.path.isdir(path):
            path = os.path.join(path, "tokenizer.model")  # tokenizer_args.h:37
        err = ctypes.create_string_buffer(512)
        self._h = lib().oracle_tik_load(path.encode(), err, 512)
        if not self._h:
            raise ValueError(err.value.decode())

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().oracle_tik_free(self._h)
                self._h = None
        except Exception:
            pass

    def vocab_size(self):
        return lib().oracle_tik_vocab_size(self._h)

    def encode(self, text: bytes):
        cap = len(text) + 8
        out = np.zeros(cap, dtype=np.int32)
        n = lib().oracle_tik_encode(self._h, text, len(text), out.ctypes.data, cap)
        return out[:n].copy()


def gpt2_bytes_to_unicode():
    """The GPT-2 byte <-> printable-char table used by HF ByteLevel (byte -> str of one char)."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(0xA1, 0xAC + 1)) + list(range(0xAE, 0xFF + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return {b: chr(c) for b, c in zip(bs, cs)}


CL100K_FAMILY = {
    r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+": 3,
    r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+": 1,
}


DEEPSEEK_V3_SPLITS = (
    r"\p{N}{1,3}", "[一-龥぀-ゟ゠-ヿ]+",
    "[!\"#$%&'()*+,\\-./:;<=>?@\\[\\\\\\]^_`{|}~][A-Za-z]+|[^\r\n\\p{L}\\p{P}\\p{S}]?[\\p{L}\\p{M}]+|"
    " ?[\\p{P}\\p{S}]+[\r\n]*|\\s*[\r\n]+|\\s+(?!\\S)|\\s+")


def hf_pattern_of(pre):
    """(pattern kind, digits) of a tokenizer.json pre_tokenizer: (1, 0) = ByteLevel with its own GPT-2 regex,
    (2, K) = Sequence[Split(cl100k-family regex, Isolated), ByteLevel(use_regex = false)]."""
    if pre["type"] == "ByteLevel":
        assert pre.get("use_regex", True) and not pre.get("add_prefix_space", False)
        return 1, 0
    assert pre["type"] == "Sequence", pre
    if len(pre["pretokenizers"]) == 4:       # DeepSeek-V3 / R1: three Isolated splits, then ByteLevel(use_regex = false)
        s1, s2, s3, bl = pre["pretokenizers"]
        for sp in (s1, s2, s3):
            assert sp["type"] == "Split" and sp["behavior"] == "Isolated" and not sp.get("invert", False)
        assert (s1["pattern"]["Regex"], s2["pattern"]["Regex"], s3["pattern"]["Regex"]) == DEEPSEEK_V3_SPLITS
        assert bl["type"] == "ByteLevel" and not bl.get("use_regex", True) and not bl.get("add_prefix_space", False)
        return 3, 3
    assert len(pre["pretokenizers"]) == 2, pre
    sp, bl = pre["pretokenizers"]
    assert sp["type"] == "Split" and sp["behavior"] == "Isolated" and not sp.get("invert", False)
    assert bl["type"] == "ByteLevel" and not bl.get("use_regex", True) and not bl.get("add_prefix_space", False)
    return 2, CL100K_FAMILY[sp["pattern"]["Regex"]]


class HfBpeOracle:
    """FastTokenizer (xllm_service/tokenizer/fast_tokenizer.cpp:20-30 over HF `tokenizers`) for byte-level BPE
    tokenizer.json files; algorithm in oracle/hf_bpe_oracle.cc, the JSON is read here."""

    def __init__(self, model_dir_or_file):
        import json
        path = model_dir_or_file
        if os.path.isdir(path):
            path = os.path.join(path, "tokenizer.json")
        with open(path, encoding="utf-8") as f:
            d = json.load(f)
        m = d["model"]
        assert m["type"] == "BPE"
        self.pattern, self.digits = hf_pattern_of(d["pre_tokenizer"])
        norm = d.get("normalizer")
        if norm == {"type": "Sequence", "normalizers": []}:   # DeepSeek-V3 ships an empty normalizer sequence
            norm = None
        assert norm is None or norm == {"type": "NFC"}, norm
        self.nfc = norm is not None
        self.ignore_merges = bool(m.get("ignore_merges", False))
        vocab = m["vocab"]
        b2u = gpt2_bytes_to_unicode()
        byte_sym = np.array([vocab[b2u[b]] for b in range(256)], dtype=np.int32)
        mg = []
        for e in m["merges"]:
            a, b = e if isinstance(e, list) else e.split(" ")
            mg.append((vocab[a], vocab[b], vocab[a + b]))
        merges = np.array(mg, dtype=np.int32).reshape(-1, 3)
        # the ids `tokenizers` gives added tokens when it loads the file (AddedVocabulary::add_tokens, in list
        # order), whatever ids the file lists: a content that is a vocabulary entry or an earlier added token keeps
        # that id, any other gets len(vocab), or one past the largest added id once that is at least len(vocab)
        given, flags, listed = {}, {}, []
        for t in d.get("added_tokens", []):
            c = t["content"]
            f = (bool(t.get("special", False)), bool(t.get("normalized", not t.get("special", False))))
            assert flags.setdefault(c, f) == f, "added token %r listed twice with different flags" % c
            if c not in given:
                listed.append(t)
                top = max(given.values(), default=None)
                given[c] = vocab[c] if c in vocab else (len(vocab) if top is None or top < len(vocab) else top + 1)
        self.added = [(t["content"], given[t["content"]], bool(t.get("special", False)),
                       bool(t.get("normalized", not t.get("special", False)))) for t in listed]
        added = [(c.encode("utf-8"), i) for c, i, _, _ in self.added]
        blob = b"".join(a for a, _ in added)
        off = np.zeros(len(added) + 1, dtype=np.int64)
        if added:
            np.cumsum([len(a) for a, _ in added], out=off[1:])
        ids = np.array([i for _, i in added], dtype=np.int32)
        norm = np.array([n for _, _, _, n in self.added] or [0], dtype=np.uint8)
        self._keep = (byte_sym, merges, blob, off, ids, norm)
        self._h = lib().oracle_hf_new(byte_sym.ctypes.data, merges.ctypes.data, merges.shape[0],
                                      ctypes.c_char_p(blob), off.ctypes.data, ids.ctypes.data, norm.ctypes.data,
                                      len(added))
        u2b = {c: b for b, c in b2u.items()}
        raw = [(bytes(u2b[ch] for ch in tok), i) for tok, i in vocab.items() if all(ch in u2b for ch in tok)]
        vblob = b"".join(r for r, _ in raw)
        voff = np.zeros(len(raw) + 1, dtype=np.int64)
        np.cumsum([len(r) for r, _ in raw], out=voff[1:])
        vids = np.array([i for _, i in raw], dtype=np.int32)
        lib().oracle_hf_configure(self._h, self.pattern, self.digits, int(self.ignore_merges), ctypes.c_char_p(vblob),
                                  voff.ctypes.data, vids.ctypes.data, len(raw))
        tp = d.get("post_processor") or {}
        procs = tp.get("processors", [tp]) if tp else []
        self.prefix_ids, self.suffix_ids = [], []
        for pr in procs:
            if pr.get("type") == "TemplateProcessing":
                seen = False
                for it in pr["single"]:
                    if "Sequence" in it:
                        seen = True
                    else:
                        (self.suffix_ids if seen else self.prefix_ids).extend(
                            pr["special_tokens"][it["SpecialToken"]["id"]]["ids"])
        self.vocab_size = max(vocab.values()) + 1
        self._vocab_id = vocab.get
        # Tokenizer::get_vocab_size(with_added_tokens = true): the vocabulary plus the added tokens it lacks
        self.vocab_size_with_added = len(vocab) + len({i for _, i, _, _ in self.added if i >= len(vocab)})
        self._token = {i: c for c, i in vocab.items()}
        self._token.update({i: c for c, i, _, _ in self.added})
        self._special = {i for _, i, s, _ in self.added if s}
        self._u2b = {c: b for b, c in b2u.items()}

    def token_to_id(self, content):
        for c, i, _, _ in self.added:
            if c == content:
                return i
        return self._vocab_id(content)

    def decode(self, ids, skip_special_tokens=False):
        """Tokenizer::decode: tokens (added ones too) through the ByteLevel decoder, each mapped back to bytes when all
        its chars are in the byte alphabet and kept verbatim otherwise, the joined bytes read as String::from_utf8_lossy
        does (Python's errors="replace" takes the same maximal subparts); unknown ids and, on request, special tokens
        are left out."""
        out = bytearray()
        for i in ids:
            t = self._token.get(int(i))
            if t is None or (skip_special_tokens and int(i) in self._special):
                continue
            if all(ch in self._u2b for ch in t):
                out += bytes(self._u2b[ch] for ch in t)
            else:
                out += t.encode("utf-8")
        return bytes(out).decode("utf-8", errors="replace")

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().oracle_hf_free(self._h)
                self._h = None
        except Exception:
            pass

    def encode(self, text: bytes):
        """ids, or None when the text is not valid UTF-8 (the reference's Rust shim panics there).  A `normalizer:
        NFC` is applied here (Python's unicodedata); template ids are NOT added (see prefix_ids / suffix_ids)."""
        if self.nfc:
            import unicodedata
            try:
                text = unicodedata.normalize("NFC", text.decode("utf-8")).encode("utf-8")
            except UnicodeDecodeError:
                return None
        cap = len(text) + 16
        out = np.zeros(cap, dtype=np.int32)
        n = lib().oracle_hf_encode(self._h, text, len(text), out.ctypes.data, cap)
        return None if n < 0 else out[:n].copy()
