"""ctypes bindings of oracle/_ref/libxllm_ref.so — the REFERENCE'S OWN hash / index / routing code compiled
unmodified (oracle/build_ref.sh, oracle/ref_shim/ref_shim.cc).  TEST INFRASTRUCTURE ONLY — see oracle/__init__.py.
`RefIndex` has the interface of oracle.PrefixOracle so the same history can be replayed on both."""
import ctypes
import os
import subprocess

import numpy as np

from .oracle import _keys_buf, _name_array

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_ref", "libxllm_ref.so")
_lib = None


def build():
    """Compile oracle/_ref from the reference checkout when that tree is present."""
    subprocess.check_call(["bash", os.path.join(_HERE, "build_ref.sh")])


def available():
    if not os.path.exists(_LIB_PATH):
        try:
            build()
        except Exception:
            return False
    return os.path.exists(_LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError("oracle/_ref/libxllm_ref.so is not built (needs the reference checkout: bash oracle/build_ref.sh)")
        L = ctypes.CDLL(_LIB_PATH)
        VP, I, SZ = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
        L.ref_xxh3_128bits_hash.argtypes = [VP, VP, SZ, ctypes.c_uint32, VP]
        L.ref_index_new.argtypes = [ctypes.c_uint32, ctypes.c_uint32, I, VP, ctypes.c_char_p]
        L.ref_index_new.restype = VP
        L.ref_index_free.argtypes = [VP]
        L.ref_index_free.restype = None
        L.ref_index_size.argtypes = [VP]
        L.ref_index_size.restype = ctypes.c_long
        L.ref_index_record.argtypes = [VP, ctypes.c_char_p, VP, SZ, VP, SZ, VP, SZ]
        L.ref_index_record.restype = None
        L.ref_index_upload.argtypes = [VP]
        L.ref_etcd_put.argtypes = [VP, VP, VP, I, VP, I, VP, I]
        L.ref_etcd_put.restype = None
        L.ref_etcd_put_raw.argtypes = [VP, ctypes.c_char_p, SZ, ctypes.c_char_p, SZ]
        L.ref_etcd_put_raw.restype = None
        L.ref_etcd_delete.argtypes = [VP, VP]
        L.ref_etcd_delete.restype = None
        L.ref_etcd_batch.argtypes = [VP, I]
        L.ref_etcd_batch.restype = None
        L.ref_etcd_list.argtypes = [VP, ctypes.c_char_p, VP, SZ, VP, SZ, VP, VP, SZ]
        L.ref_etcd_list.restype = ctypes.c_long
        L.ref_index_get.argtypes = [VP, VP, VP, I, VP]
        L.ref_index_match.argtypes = [VP, VP, SZ, VP, I, VP, VP, VP, VP]
        L.ref_index_match.restype = None
        L.ref_registry_set_instance.argtypes = [VP, ctypes.c_char_p, I, I]
        L.ref_registry_set_instance.restype = None
        L.ref_registry_set_load.argtypes = [VP, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_float]
        L.ref_registry_set_load.restype = None
        L.ref_registry_clear_load.argtypes = [VP, ctypes.c_char_p]
        L.ref_registry_clear_load.restype = None
        L.ref_route_car.argtypes = [VP, VP, SZ, VP, I, VP, VP]
        _lib = L
    return _lib


def xxh3_128bits_hash(prev, token_ids, seed=1024) -> bytes:
    """The reference's common/hash_util.cpp:18-45 itself (CHECK-aborts when 4*n + 16 >= 1024, like the reference)."""
    t = np.ascontiguousarray(token_ids, dtype=np.int32)
    out = ctypes.create_string_buffer(16)
    pbuf = ctypes.create_string_buffer(bytes(prev), 16) if prev is not None else None
    lib().ref_xxh3_128bits_hash(pbuf, t.ctypes.data, t.size, seed, out)
    return out.raw


def block_hash_chain(token_ids, block_size=128, seed=1024) -> np.ndarray:
    """The chain loop of GlobalKVCacheMgr::match (global_kvcache_mgr.cpp:85-94) over ref xxh3_128bits_hash."""
    t = np.ascontiguousarray(token_ids, dtype=np.int32)
    nb = t.size // block_size
    keys = np.zeros((nb, 16), dtype=np.uint8)
    prev = None
    for b in range(nb):
        prev = xxh3_128bits_hash(prev, t[b * block_size:(b + 1) * block_size], seed)
        keys[b] = np.frombuffer(prev, np.uint8)
    return keys


class RefIndex:
    """GlobalKVCacheMgr + InstanceMgr::get_load_metrics + CacheAwareRouting — the reference's classes — on an
    in-memory etcd.  master=False with share=<a master RefIndex> gives a replica fed by the etcd watch."""
    DEFAULT, PREFILL, DECODE, MIX = 0, 1, 2, 3

    def __init__(self, names, block_size=128, seed=1024, master=True, share=None, namespace=""):
        self.names = list(names)
        self._names = _name_array(self.names)
        self.block_size, self.seed = block_size, seed
        self._h = lib().ref_index_new(block_size, seed, int(master), share._h if share is not None else None,
                                      namespace.encode())

    def __del__(self):
        try:
            if self._h:
                lib().ref_index_free(self._h)
                self._h = None
        except Exception:
            pass

    def record(self, name, stored=(), offload=(), removed=()):
        s, ns = _keys_buf(stored)
        o, no = _keys_buf(offload)
        r, nr = _keys_buf(removed)
        lib().ref_index_record(self._h, name.encode(), s.ctypes.data, ns, o.ctypes.data, no, r.ctypes.data, nr)

    def upload(self):
        return bool(lib().ref_index_upload(self._h))

    def put(self, key, hbm=(), dram=(), ssd=()):
        """an etcd PUT of this key's CacheLocations (DELETE when all three sets are empty: etcd_client.cpp:131-133)"""
        k = np.ascontiguousarray(np.frombuffer(bytes(key), dtype=np.uint8))
        lib().ref_etcd_put(self._h, k.ctypes.data, _name_array(list(hbm)), len(hbm), _name_array(list(dram)),
                           len(dram), _name_array(list(ssd)), len(ssd))

    def put_raw(self, key: bytes, value: bytes):
        lib().ref_etcd_put_raw(self._h, key, len(key), value, len(value))

    def delete(self, key):
        k = np.ascontiguousarray(np.frombuffer(bytes(key), dtype=np.uint8))
        lib().ref_etcd_delete(self._h, k.ctypes.data)

    def batch(self, begin: bool):
        lib().ref_etcd_batch(self._h, int(begin))

    def etcd_pairs(self, prefix=b"XLLM:CACHE:"):
        """[(key bytes, value bytes)] currently in the store under prefix (namespace included by the caller)."""
        kcap, vcap, mp = 1 << 16, 1 << 20, 1 << 10
        while True:
            kb, vb = ctypes.create_string_buffer(kcap), ctypes.create_string_buffer(vcap)
            kl, vl = np.zeros(mp, np.int64), np.zeros(mp, np.int64)
            n = lib().ref_etcd_list(self._h, prefix, kb, kcap, vb, vcap, kl.ctypes.data, vl.ctypes.data, mp)
            if n >= 0:
                break
            kcap, vcap, mp = kcap * 4, vcap * 4, max(mp * 4, -n)
        out, ko, vo = [], 0, 0
        for i in range(n):
            out.append((kb.raw[ko:ko + kl[i]], vb.raw[vo:vo + vl[i]]))
            ko += int(kl[i])
            vo += int(vl[i])
        return out

    def size(self):
        return lib().ref_index_size(self._h)

    def get(self, key):
        k = np.ascontiguousarray(np.frombuffer(bytes(key), dtype=np.uint8))
        m = np.zeros(3, dtype=np.uint64)
        found = lib().ref_index_get(self._h, k.ctypes.data, self._names, len(self.names), m.ctypes.data)
        return bool(found), [int(x) for x in m]

    def set_instance(self, name, type_, schedulable=True):
        lib().ref_registry_set_instance(self._h, name.encode(), type_, int(schedulable))

    def set_load(self, name, waiting, usage):
        lib().ref_registry_set_load(self._h, name.encode(), int(waiting), float(usage))

    def clear_load(self, name):
        lib().ref_registry_clear_load(self._h, name.encode())

    def match(self, tokens):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        n = len(self.names)
        scores = np.zeros((3, n), dtype=np.uint32)
        inst = ctypes.c_uint64()
        mb, mm = ctypes.c_uint32(), ctypes.c_uint32()
        lib().ref_index_match(self._h, t.ctypes.data, t.size, self._names, n, scores.ctypes.data, ctypes.byref(inst),
                              ctypes.byref(mb), ctypes.byref(mm))
        return {"hbm": scores[0], "dram": scores[1], "ssd": scores[2], "instances": inst.value,
                "max_block_num": mb.value, "max_matched_block_num": mm.value}

    def route(self, tokens):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        pid, did = ctypes.c_int(), ctypes.c_int()
        ok = lib().ref_route_car(self._h, t.ctypes.data, t.size, self._names, len(self.names), ctypes.byref(pid),
                                 ctypes.byref(did))
        return {"ok": bool(ok), "prefill_id": pid.value, "decode_id": did.value}
