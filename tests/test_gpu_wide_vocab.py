"""The tokenizer kernels at token ids and merge ranks past 65 535 (the wide, non-SMALL instantiations: 32-bit pair
state, 28-bit memo ids, 4 ids per memo entry) on the SentencePiece BPE, SentencePiece Unigram and tiktoken backends.

The models are the committed ones with ~70 000 filler pieces spliced in front of their real pieces
(tests/golden/make_wide_fixtures.py): every real id moves up by the filler count, and nothing else changes, so the
committed upstream goldens, mapped, are an exact reference.  The derived models are rebuilt here from the committed
files; their SHA-256 is checked against the one frozen next to goldens that upstream produced on them
(tests/golden/wide_goldens.json).  The first tests run without a GPU; the rest are marked gpu."""
import hashlib
import importlib.util
import json
import os
import random

import numpy as np
import pytest

HERE = os.path.dirname(__file__)
GOLD = os.path.join(HERE, "golden", "wide_goldens.json")
WIDE = ["sp_bpe_8k", "sp_natural_32k", "sp_unigram_4k", "sp_unigram_4k_bf", "tiktoken_1k"]
BOUNDARY = ["sp_bpe_8k@65534", "sp_bpe_8k@65535", "sp_bpe_8k@65536"]


def _load_generator():
    spec = importlib.util.spec_from_file_location("make_wide_fixtures", os.path.join(HERE, "golden", "make_wide_fixtures.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


MW = _load_generator()

# The encode variants of test_gpu_memo.py.  On a Unigram model every one of them runs the same kernel (Unigram has no
# word memo, no warm-up kernels and no express kernel: the result of a word depends on the running score), and the
# tiktoken backend has no express kernel (byte mode); they still run, to show the knobs leave those backends exact.
VARIANTS = [
    ("default", {}),                                  # express kernel + memo
    ("memo_off", {"XLLM_SP_MEMO_SLOTS": "0"}),
    ("memo_4", {"XLLM_SP_MEMO_SLOTS": "4"}),          # nearly every insert fails
    ("warm", {"XLLM_SP_WARM": "1"}),
    ("express_off", {"XLLM_SP_EXPRESS": "0"}),        # every window takes the buffer path
]


class Derived:
    def __init__(self, name, root):
        self.name, self.base = name, MW.DERIVED[name][0]
        self.dir = str(root / name.replace("@", "_"))
        self.first, self.n_fill, model = MW.write_derived(name, self.dir)
        self.sha256 = hashlib.sha256(model).hexdigest()
        self.base_dir = os.path.join(HERE, "golden", self.base)
        self.tiktoken = self.base.startswith("tiktoken")

    def map(self, ids):
        return MW.map_ids(list(ids), self.first, self.n_fill)

    def oracle(self, o):
        return o.TiktokenOracle(self.dir) if self.tiktoken else o.SentencePieceOracle(self.dir)


@pytest.fixture(scope="module")
def gold():
    with open(GOLD) as f:
        return json.load(f)["models"]


@pytest.fixture(scope="module")
def derived(tmp_path_factory):
    root = tmp_path_factory.mktemp("wide_models")
    return {name: Derived(name, root) for name in MW.DERIVED}


def _handle(model_dir, env=None):
    import xllm_service_b200 as x
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return x.Ingest(tokenizer_path=model_dir)   # the knobs are read when the handle is created
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def _encode(h, texts, stride):
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    return h.encode_batch(b.text, b.offsets, stride)


def _check(h, texts, want, stride=None):
    """ids, n_ids and status of every row against the expected id lists; a row the stride truncates holds the
    expected prefix, with the full count and status 1."""
    if stride is None:
        stride = max(16, max((len(w) for w in want), default=0) + 8)
    ids, n_ids, status = _encode(h, texts, stride)
    bad = []
    for i, w in enumerate(want):
        keep = min(len(w), stride)
        if int(n_ids[i]) != len(w) or int(status[i]) != (1 if len(w) > stride else 0) or ids[i, :keep].tolist() != w[:keep]:
            bad.append((i, texts[i][:40], int(n_ids[i]), len(w), int(status[i])))
    assert not bad, (len(bad), bad[:4])
    return ids, n_ids, status


def _mix(seed, n=160):
    """Heavy word repetition across and inside prompts (the memo's hit path), words at and past the 15-byte memo key,
    words with more ids than a memo entry holds, unknown chars, bare U+2581 words, doubled spaces."""
    from xllm_service_b200 import workload
    rnd = random.Random(seed)
    vocab = [w.decode() for w in workload.make_vocabulary()[:300]]
    odd = ["a" * 14, "b" * 15, "c" * 16, "d" * 17, "zqxjkvwpyfgh", "zqxjkvwpyfghmn", "日本", "é", "naïve", "x1y2z3",
           "▁", "▁▁", "don't", "\x00", "ÿ", "🙂", "12345678901234", "Zq" * 7, "zq" * 8, "v", "vv"]
    out = []
    for _ in range(n):
        words = []
        for _ in range(rnd.randrange(1, 400)):
            words.append(rnd.choice(odd) if rnd.random() < 0.15 else rnd.choice(vocab))
            if rnd.random() < 0.05:
                words.append("")
        out.append(" ".join(words).encode())
    return out + [b"", b" ", b"same same same same same same same same", ("word " * 3000).encode()]


# ---------------------------------------------------------------------------- without a GPU
@pytest.mark.parametrize("name", list(MW.DERIVED))
def test_derived_model_is_the_one_upstream_ran(derived, gold, name):
    d, g = derived[name], gold[name]
    assert d.sha256 == g["sha256"]
    assert (d.first, d.n_fill) == (g["first_shifted"], g["n_fill"])
    from xllm_service_b200 import _lib
    base = _lib.tokenizer_probe(d.base_dir)["n_pieces"]
    info = _lib.tokenizer_probe(d.dir)
    assert info["n_pieces"] == base + d.n_fill == g["n_pieces"]


@pytest.mark.parametrize("name", list(MW.DERIVED))
def test_oracle_on_derived_model(oracle, derived, gold, name):
    """The project's CPU oracle on the derived model equals the committed goldens, mapped, and the goldens upstream
    produced on the derived model itself."""
    d = derived[name]
    orc = d.oracle(oracle)
    bad = [t[:40] for t, ids in MW.committed_goldens(d.base) if orc.encode(t).tolist() != d.map(ids)]
    assert not bad, (len(bad), bad[:3])
    cases = gold[name]["cases"]
    bad = [c["text"][:40] for c in cases if orc.encode(bytes.fromhex(c["text"])).tolist() != c["ids"]]
    assert not bad, (len(bad), bad[:3])
    assert max(max(c["ids"], default=0) for c in cases) >= 65533


# ---------------------------------------------------------------------------- GPU: each backend, each variant
@pytest.mark.gpu
@pytest.mark.parametrize("variant,env", VARIANTS, ids=[v[0] for v in VARIANTS])
@pytest.mark.parametrize("name", WIDE)
def test_backend_vs_mapped_goldens_and_oracle(oracle, derived, gold, name, variant, env):
    d = derived[name]
    texts, want = [], []
    for t, ids in MW.committed_goldens(d.base):
        texts.append(t)
        want.append(d.map(ids))
    for c in gold[name]["cases"]:
        texts.append(bytes.fromhex(c["text"]))
        want.append(c["ids"])
    orc = d.oracle(oracle)
    fuzz = _mix(31)
    texts += fuzz
    want += [orc.encode(t).tolist() for t in fuzz]
    assert max(max(w, default=0) for w in want) > 65535
    h = _handle(d.dir, env)
    try:
        for _ in range(2):                      # a second launch: the memo starts empty again
            _check(h, texts, want)
    finally:
        h.close()


# ---------------------------------------------------------------------------- GPU: memo payloads in the wide format
@pytest.mark.gpu
@pytest.mark.parametrize("variant,env", [VARIANTS[0], VARIANTS[3], VARIANTS[4]], ids=["default", "warm", "express_off"])
def test_memo_payload_edges(oracle, derived, variant, env):
    """A wide memo entry holds at most 4 ids of 28 bits: words of exactly 1, 4 and 5 ids (the last one never fits),
    and words of 15 (the longest key) and 16 key bytes, each repeated often enough to be inserted and hit both in the
    express kernel and on the buffer path."""
    from xllm_service_b200 import workload
    d = derived["sp_bpe_8k"]
    orc = d.oracle(oracle)
    vocab = [w.decode() for w in workload.make_vocabulary()[:4000]]
    by_n = {}
    for w in vocab:
        by_n.setdefault(len(orc.encode(w.encode())), []).append(w)
    rnd = random.Random(5)
    keyed = {15: [], 16: []}                    # two or three one-id words glued into 15 / 16 key bytes
    while min(len(v) for v in keyed.values()) < 16:
        w = "".join(rnd.choice(by_n[1]) for _ in range(rnd.choice((2, 3))))
        if len(w) in keyed and len(keyed[len(w)]) < 16:
            keyed[len(w)].append(w)
    n15 = {len(orc.encode(w.encode())) for w in keyed[15]}
    assert {1, 4, 5} <= set(by_n) and min(n15) <= 4 < max(n15), (sorted(by_n), n15)   # some 15-byte words fit, some not
    pool = by_n[1][:20] + by_n[4][:20] + by_n[5][:20] + keyed[15] + keyed[16]
    texts = []
    for i in range(300):
        words = [rnd.choice(pool) for _ in range(rnd.randrange(1, 200))]
        if i % 3 == 0:
            words = [rnd.choice(pool)] * rnd.randrange(2, 90)   # one word over and over: hits within a window
        texts.append(" ".join(words).encode())
    want = [orc.encode(t).tolist() for t in texts]
    assert all(i > 65535 for i in orc.encode(" ".join(by_n[1][:20]).encode()).tolist())
    h = _handle(d.dir, env)
    try:
        _check(h, texts, want)
    finally:
        h.close()


# ---------------------------------------------------------------------------- GPU: express-kernel seams at wide ids
def _words(rnd, n, lo=1, hi=9, alphabet="abcdefghijklmnopqrstuvwxyz"):
    return ["".join(rnd.choice(alphabet) for _ in range(rnd.randint(lo, hi))) for _ in range(n)]


def _text(rnd, nbytes):
    out, size = [], 0
    while size < nbytes:
        w = _words(rnd, 1, 1, 9)[0]
        out.append(w)
        size += len(w) + 1
    return " ".join(out).encode()[:nbytes]


def _seam_texts():
    rnd = random.Random(3)
    # more than 64 words in one 512-byte window
    texts = [b"a " * 400, b"a b " * 200 + b"cd", b"ab " * 600, b"a  b   c    d " * 80, (b"i " * 63 + b"longerword ") * 12,
             (b"v " * 65 + b"x") * 6]
    for n in (63, 64, 65, 66, 127, 128, 129):
        texts.append(" ".join(_words(rnd, n, 1, 3)).encode())
    # every word length 1..15 at every start offset mod 16, in the first window and past 256 / 480 bytes
    for n in range(1, 16):
        for off in range(16):
            w = "".join(rnd.choice("abcdefghijklmnopv") for _ in range(n))
            for lead in (off, 256 + off, 480 + off):
                head = "".join(rnd.choice("xy ") for _ in range(lead - 1)) + " " if lead else ""
                texts.append((head + w + " " + w + " tail").encode())
    # a long or hard word (over 15 bytes, or more ids than a wide memo entry holds) as word 30..97 of a run
    odd = ["".join(rnd.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(n)) for n in (16, 17, 24, 40)]
    odd += ["{}[]{}[]{}[]{}", "~`~`~`~`~`~`~`", "qzxjvkqzxjvkqzx", "Q9z~X8y`W7v^U6t", "qzxjv", "日本語"]
    for k in list(range(30, 68)) + [95, 96, 97]:
        for o in odd:
            texts.append((" ".join(_words(rnd, k, 1, 4)) + " " + o + " " + " ".join(_words(rnd, 80, 1, 6))).encode())
    return texts


@pytest.mark.gpu
def test_express_seams(oracle, derived):
    d = derived["sp_bpe_8k"]
    orc = d.oracle(oracle)
    texts = _seam_texts()
    h = _handle(d.dir)
    try:
        _check(h, texts, [orc.encode(t).tolist() for t in texts])
        # a truncating ids_stride in some requests only: every fourth one is far longer than the row
        rnd = random.Random(17)
        texts = [_text(rnd, 3000 + 37 * i) if i % 4 == 1 else _text(rnd, rnd.randint(0, 80)) for i in range(60)]
        _, _, status = _check(h, texts, [orc.encode(t).tolist() for t in texts], stride=96)
        assert (status == 1).sum() >= 12 and (status == 0).sum() >= 12
    finally:
        h.close()


# ---------------------------------------------------------------------------- GPU: the narrow / wide boundary
@pytest.mark.gpu
@pytest.mark.parametrize("name", BOUNDARY)
def test_narrow_wide_boundary(oracle, derived, gold, name):
    """65 534 pieces: the last model on the 16-bit kernels (top id 65 533); 65 535: the first on the wide kernels (top
    id 65 534); 65 536: the first whose ids do not all fit a uint16.  The real pieces hold the top ids, and the frozen
    texts produce the top one.  ids_u16 equals the int32 download while every id fits, and is refused past that."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    d = derived[name]
    g = gold[name]
    top = g["n_pieces"] - 1
    texts = [bytes.fromhex(c["text"]) for c in g["cases"]]
    want = [c["ids"] for c in g["cases"]]
    assert any(top in w for w in want)
    for t, ids in MW.committed_goldens(d.base):
        texts.append(t)
        want.append(d.map(ids))
    for variant, env in (VARIANTS[0], VARIANTS[4]):
        h = _handle(d.dir, env)
        try:
            _check(h, texts, want)
        finally:
            h.close()
    b = workload.pack_prompts(texts)
    h = x.Ingest(tokenizer_path=d.dir)
    try:
        a = h.ingest_batch(b.text, b.offsets, 256, want_match=False)
        assert (a["status"] <= 1).all() and a["ids"].max() == top
        if g["n_pieces"] <= 65535:
            c = h.ingest_batch(b.text, b.offsets, 256, want_match=False, ids_u16=True)
            assert c["ids"].dtype == np.uint16
            assert (c["ids"].astype(np.int32) == a["ids"]).all()
            for f in ("n_ids", "status", "keys"):
                assert (a[f] == c[f]).all(), f
        else:
            with pytest.raises(x.IngestError) as e:
                h.ingest_batch(b.text, b.offsets, 256, want_match=False, ids_u16=True)
            assert e.value.code == -5     # XLLM_ERR_UNSUPPORTED
    finally:
        h.close()


@pytest.mark.gpu
def test_narrow_download_refused_far_past_16_bits(derived):
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    for name in WIDE:
        b = workload.pack_prompts([b"hello world"])
        h = x.Ingest(tokenizer_path=derived[name].dir)
        try:
            with pytest.raises(x.IngestError) as e:
                h.ingest_batch(b.text, b.offsets, 64, want_match=False, ids_u16=True)
            assert e.value.code == -5, name
        finally:
            h.close()


# ---------------------------------------------------------------------------- GPU: the whole ingest path
@pytest.mark.gpu
@pytest.mark.parametrize("name", WIDE)
def test_ingest_keys_hash_wide_ids(oracle, derived, name):
    """Block keys are the chained hash of the full 32-bit ids: ids past 65 535 reach the hash unmasked."""
    from xllm_service_b200 import workload
    d = derived[name]
    orc = d.oracle(oracle)
    texts = [s.encode() for s in workload.sentences(300, (5, 300), seed=23)] + [b"", b"v " * 200]
    b = workload.pack_prompts(texts)
    T = 1024
    h = _handle(d.dir)
    try:
        h.set_pipeline(37, 1 << 20)
        out = h.ingest_batch(b.text, b.offsets, T, want_match=False)
    finally:
        h.close()
    n_blocks = 0
    for r, t in enumerate(texts):
        want = orc.encode(t)
        n = min(want.size, T)
        assert out["n_ids"][r] == want.size and out["status"][r] == (1 if want.size > T else 0), r
        assert (out["ids"][r, :n] == want[:n]).all(), r
        keys = oracle.block_hash_chain(want[:n])
        assert (out["keys"][r, :keys.shape[0]] == keys).all(), r
        assert not out["keys"][r, keys.shape[0]:].any(), r
        n_blocks += keys.shape[0]
    assert n_blocks > 200 and out["ids"].max() > 65535


@pytest.mark.gpu
def test_segments_with_wide_ids(oracle, derived):
    """xllm_ingest_batch_segments: text pieces encoded like separate calls, id spans (here past 65 535 too) copied."""
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    d = derived["sp_bpe_8k"]
    orc = d.oracle(oracle)
    rnd = random.Random(29)
    reqs = [
        [b"hello world, plain text", np.arange(70000, 70300, dtype=np.int32), " ".join(_words(rnd, 200)).encode()],
        [np.full(130, 0x0FFFFFFF, np.int32), b"v v v"],
        [b"", np.arange(65530, 65542, dtype=np.int32), b"", "café naïve 日本".encode()],
        [" ".join(_words(rnd, 150)).encode()],
        [np.array([77999, 65535, 65536, 131071], np.int32), b" tail words", np.array([1 << 27], np.int32)],
    ]
    pieces, seg_len, spans, rss = [], [], [], [0]
    for r in reqs:
        for s in r:
            if isinstance(s, bytes):
                pieces.append(s)
                seg_len.append(-1)
            else:
                spans.append(s)
                seg_len.append(s.size)
        rss.append(len(seg_len))
    pb = workload.pack_prompts(pieces)
    b = workload.SegmentBatch(pb.text, pb.offsets, np.asarray(rss, np.int32), np.asarray(seg_len, np.int32),
                              np.concatenate(spans).astype(np.int32), np.zeros(len(reqs), bool),
                              np.zeros(len(reqs), np.int32))
    T = 2048
    h = x.Ingest(tokenizer_path=d.dir)
    try:
        out = h.ingest_batch_segments(b, T, want_match=False)
    finally:
        h.close()
    for r, segs in enumerate(reqs):
        want = np.concatenate([orc.encode(s) if isinstance(s, bytes) else s for s in segs]).astype(np.int32)
        assert out["status"][r] == 0 and out["n_ids"][r] == want.size, r
        assert (out["ids"][r, :want.size] == want).all(), r
        keys = oracle.block_hash_chain(want)
        assert (out["keys"][r, :keys.shape[0]] == keys).all(), r


# ---------------------------------------------------------------------------- GPU: metamorphic bulk check
@pytest.mark.gpu
@pytest.mark.parametrize("name", WIDE)
def test_derived_equals_mapped_committed(derived, name):
    """~4 096 mixed prompts: the GPU result on the derived model equals the GPU result on the committed model, mapped.
    Both sides run the same tokenization logic; only the id width differs."""
    from xllm_service_b200 import workload
    d = derived[name]
    texts = [s.encode() for s in workload.sentences(3900, (1, 60), seed=43)] + _mix(47, 190)
    assert len(texts) >= 4090
    stride = max(16, 3 * max(len(t) for t in texts) + 8)
    res = []
    for model in (d.base_dir, d.dir):
        h = _handle(model)
        try:
            res.append(_encode(h, texts, stride))
        finally:
            h.close()
    (i0, n0, s0), (i1, n1, s1) = res
    assert (s0 == 0).all() and (s1 == 0).all()
    assert (n0 == n1).all()
    valid = np.arange(stride)[None, :] < n0[:, None]
    mapped = np.where(i0 >= d.first, i0 + d.n_fill, i0)
    assert (i1[valid] == mapped[valid]).all()
    assert i1[valid].max() > 65535
