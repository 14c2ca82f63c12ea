"""Rows a5-a8 / f1 / f3 pinned to the REFERENCE ITSELF: oracle/_ref/libxllm_ref.so is the reference's own
hash_util.cpp, types.h, global_kvcache_mgr.cpp, etcd_client.cpp, cache_aware_routing.cpp and
InstanceMgr::get_load_metrics compiled unmodified from the reference checkout (oracle/build_ref.sh) over an in-memory etcd.
The restatement (oracle/prefix_oracle.cc, oracle/xxh3_oracle.c) — which every GPU parity test compares the device
against — must agree with it on the XXH3 known answers, on random block hashes, and on random
event / upload / match / route histories.  Skipped only where neither the reference checkout nor a prebuilt _ref exists."""
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import ref

HERE = os.path.dirname(__file__)
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.skipif(not ref.available(), reason="oracle/_ref not built and the reference checkout absent")


def test_xxh3_known_answers_and_random_blocks(oracle):
    # SURVEY.md §8c KAT (libxxhash 0.8.2): tokens 0..255, block 128, seed 1024
    k = ref.block_hash_chain(np.arange(256, dtype=np.int32), 128, 1024)
    assert bytes(k[0]).hex() == "a6c0e2fc92c32b1c1ccff29b710ca0d2"
    assert bytes(k[1]).hex() == "f981264b143b2d5f81fd86ed5d58d2a1"
    assert ref.xxh3_128bits_hash(None, np.arange(16, dtype=np.int32), 1024).hex() == "1247ae96b541bccd1d2bea48ea0a97e4"
    # the chained golden vectors minted from libxxhash
    kat = json.load(open(os.path.join(HERE, "golden", "xxh3_kat.json")))
    n_chain = 0
    for c in kat.get("chains", []):
        toks = np.array(c["tokens"], dtype=np.int32) if "tokens" in c else None
        if toks is None or 4 * c["block_size"] + 16 >= 1024:
            continue
        got = ref.block_hash_chain(toks, c["block_size"], c["seed"])
        assert [bytes(x).hex() for x in got] == c["keys"]
        n_chain += 1
    # every length the reference accepts (4n + 16 < 1024, hash_util.cpp:33), chained and unchained, three seeds
    rng = np.random.default_rng(5)
    for n in list(range(0, 252)) + [128] * 50:
        for seed in (1024, 0, 0xFFFFFFFF):
            t = rng.integers(-2**31, 2**31, size=n, dtype=np.int64).astype(np.int32)
            prev = bytes(rng.integers(0, 256, 16, dtype=np.uint8)) if rng.random() < 0.7 else None
            assert ref.xxh3_128bits_hash(prev, t, seed) == oracle.xxh3_128bits_hash(prev, t, seed), (n, seed)


def _pair(oracle, names, types, block_size=128, seed=1024):
    R = ref.RefIndex(names, block_size, seed)
    P = oracle.PrefixOracle(names, block_size, seed)
    for X in (R, P):
        for n, t in zip(names, types):
            X.set_instance(n, t)
    return R, P


def _reference_survives(oracle, P, toks, bs):
    """GlobalKVCacheMgr::match dereferences hbm_instance_set.begin() inside its DRAM and SSD branches
    (global_kvcache_mgr.cpp:113-114,123-124): a matched block held only in DRAM / SSD is undefined behaviour there
    (a null-node read: the compiled reference segfaults).  Such requests can only be checked on the restatement."""
    for k in oracle.block_hash_chain(toks, bs, 1024):
        found, m = P.get(k)
        if not found or not any(m):
            return True
        if m[0] == 0:
            return False
    return True


def _same_match(a, b):
    for f in ("hbm", "dram", "ssd"):
        assert a[f].tolist() == b[f].tolist(), f
    for f in ("instances", "max_block_num", "max_matched_block_num"):
        assert a[f] == b[f], f


@pytest.mark.parametrize("seed", range(8))
def test_random_histories_oracle_equals_reference(oracle, seed):
    """Per seed: 150 independent histories x ~70 steps (~10 K operations): random KvCacheEvents
    (stored / offload / removed, several keys each) from random instances, uploads at random points, load-metric and
    schedulability changes, then match + route of prompts built to share prefixes with the indexed blocks.  After
    every upload the whole key universe is compared; every match is compared field by field; every routing decision
    must be the oracle's literal choice (same containers, same insertion history => same iteration order) and lie in
    the oracle's arg-max set."""
    rng = np.random.default_rng(1000 + seed)
    n_ops = n_ub = 0
    for hist in range(150):
        n_inst = int(rng.integers(1, 13))
        names = ["inst-%d-%d" % (hist, i) for i in range(n_inst)]
        types = [int(rng.integers(0, 4)) for _ in names]
        bs = int(rng.choice([128, 16, 64, 251, 1]))
        R, P = _pair(oracle, names, types, bs, 1024)
        # a few prompts; the key universe = their block keys + some foreign keys
        prompts = []
        for _ in range(4):
            nb = int(rng.integers(0, 9))
            tail = int(rng.integers(0, bs))
            prompts.append(rng.integers(0, 32000, nb * bs + tail).astype(np.int32))
        prompts.append(np.concatenate([prompts[0][:2 * bs], rng.integers(0, 32000, 3 * bs).astype(np.int32)]))
        universe = [oracle.block_hash_chain(p, bs, 1024) for p in prompts]
        universe = np.concatenate(universe + [rng.integers(0, 256, (4, 16), dtype=np.uint8)])
        for n in names:
            if rng.random() < 0.85:
                w, u = int(rng.integers(0, 6)), float(np.float32(rng.choice([0.0, 0.25, 0.5, 0.99, 1.0, rng.random()])))
                R.set_load(n, w, u)
                P.set_load(n, w, u)
        for step in range(int(rng.integers(40, 100))):
            op = rng.random()
            n_ops += 1
            if op < 0.45 and len(universe):
                name = names[int(rng.integers(0, n_inst))]
                pick = lambda: universe[rng.integers(0, len(universe), int(rng.integers(0, 5)))]
                kind = rng.random()
                s = pick() if kind < 0.6 else ()
                o = pick() if 0.4 < kind < 0.9 else ()
                r = pick() if kind > 0.8 else ()
                R.record(name, s, o, r)
                P.record(name, s, o, r)
            elif op < 0.6:
                assert R.upload()
                P.upload()
                assert R.size() == P.size()
                for k in universe:
                    assert R.get(k) == P.get(k)
            elif op < 0.7:
                n = names[int(rng.integers(0, n_inst))]
                if rng.random() < 0.3:
                    R.clear_load(n)
                    P.clear_load(n)
                elif rng.random() < 0.3:
                    t, sch = int(rng.integers(0, 4)), bool(rng.random() < 0.7)
                    R.set_instance(n, t, sch)
                    P.set_instance(n, t, sch)
                else:
                    w, u = int(rng.integers(0, 6)), float(np.float32(rng.random()))
                    R.set_load(n, w, u)
                    P.set_load(n, w, u)
            else:
                toks = prompts[int(rng.integers(0, len(prompts)))]
                if rng.random() < 0.2:
                    toks = toks[:int(rng.integers(0, toks.size + 1))]
                if not _reference_survives(oracle, P, toks, bs):
                    n_ub += 1
                    continue
                _same_match(R.match(toks), P.match(toks))
                a, b = R.route(toks), P.route(toks)
                assert a["ok"] == b["ok"]
                if a["ok"]:
                    assert a["prefill_id"] == b["prefill_id"] and a["decode_id"] == b["decode_id"]
                    if a["prefill_id"] >= 0:     # -1: every candidate scored <= MIN_SCORE, the name stays empty (:65,80)
                        assert (b["prefill_argmax"] >> a["prefill_id"]) & 1
                    if a["decode_id"] >= 0:
                        assert (b["decode_argmax"] >> a["decode_id"]) & 1
    assert n_ops > 9000 and n_ub < n_ops // 10


def test_replica_watch_path_oracle_equals_reference(oracle):
    """update_kvcache (global_kvcache_mgr.cpp:133-175): a replica follows a master through etcd PUT / DELETE events —
    one watch response per upload, PUTs before DELETEs, last value wins — and ends with the master's map; the oracle's
    put / delete replay of the same listing gives the same map."""
    rng = np.random.default_rng(3)
    names = ["n%d" % i for i in range(10)]
    M = ref.RefIndex(names)
    Rp = ref.RefIndex(names, master=False, share=M)
    P = oracle.PrefixOracle(names)
    keys = rng.integers(0, 256, (200, 16), dtype=np.uint8)
    for rnd in range(12):
        for _ in range(150):
            n = names[int(rng.integers(0, 10))]
            k = keys[rng.integers(0, 200, int(rng.integers(1, 4)))]
            kind = rng.random()
            args = (k, (), ()) if kind < 0.5 else ((), k, ()) if kind < 0.8 else ((), (), k)
            M.record(n, *args)
            P.record(n, *args)
        assert M.upload()
        P.upload()
        assert M.size() == Rp.size() == P.size()
        for k in keys:
            assert M.get(k) == Rp.get(k) == P.get(k)
    # one response carrying a PUT and a DELETE of the same key: the DELETE is applied last (:163-172)
    k = keys[0]
    Rp.batch(True)
    Rp.delete(k)
    Rp.put(k, hbm=["n1"])
    Rp.batch(False)
    assert Rp.get(k)[0] is False
    # an unparsable value is skipped (:149-152), a parsable one with extra keys is taken
    Rp.put_raw(b"XLLM:CACHE:" + bytes(keys[1]), b"{not json")
    assert Rp.get(keys[1]) == M.get(keys[1])
    Rp.put_raw(b"XLLM:CACHE:" + bytes(keys[1]),
               b'{"ssd_instance_set":["n3"],"x":1,"hbm_instance_set":[],"dram_instance_set":["n2","n2"]}')
    assert Rp.get(keys[1]) == (True, [0, 4, 8])


def test_index_wire_form_against_the_reference(tmp_path):
    """host/index_wire.h both ways against the reference's own etcd writer / reader (tests/cpp/index_wire_ref_main.cc)."""
    exe = tmp_path / "index_wire_ref_main"
    so = os.path.join(ROOT, "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(HERE, "cpp", "index_wire_ref_main.cc"), "-o", str(exe),
                           os.path.join(so, "libxllm_ref.so"), "-Wl,-rpath," + so])
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout[-2000:]
