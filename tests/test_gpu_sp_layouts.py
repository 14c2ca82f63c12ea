"""The SentencePiece kernels on the model layouts of tests/golden/make_sp_layouts_fixture.py, bit-exact against the
goldens upstream libsentencepiece produced and against the CPU oracle, through the C-ABI:

  llama_bpe      identity normaliser, kept whitespace, U+2581-run pieces (split_mode 2), byte fallback: the word-start
                 rule for runs of U+2581, no trailing-space strip, LF / tab / CR / NUL as byte pieces, an empty
                 normaliser trie
  nodummy_bpe    no dummy prefix (split_mode 1): the express kernel without a pending U+2581, and its hand-over
  ws_unigram     Unigram with kept whitespace (split_mode 2): words led by a U+2581 run, the running score carried
                 across them; a word of more than 511 bytes is refused with XLLM_ERR_CAPACITY (-6)
  nosplit_bpe    cross-word BPE pieces (split_mode 0): the whole prompt is one pre-token, cooperative merge then the
                 long-word kernel, many requests competing for its scratch slots
  chain_unigram  more than 32 pieces at one start and pieces of 33..64 bytes: the per-end Viterbi fallback, with
                 exact float32 ties kept on the first candidate as upstream does"""
import hashlib
import importlib.util
import json
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
GOLD = os.path.join(HERE, "golden", "sp_layouts_goldens.json")
SP = "▁".encode()
ERR_CAPACITY = -6
UNI_MAX_WORD = 511     # bytes of one Unigram word the device lattice holds


def _load_generator():
    spec = importlib.util.spec_from_file_location("make_sp_layouts_fixture",
                                                  os.path.join(HERE, "golden", "make_sp_layouts_fixture.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


ML = _load_generator()
UNIGRAM = ("ws_unigram", "chain_unigram")
BPE = [n for n in ML.NAMES if n not in UNIGRAM]

VARIANTS = [
    ("default", {}),                                  # express kernel (split_mode 1 models) + memo
    ("express_off", {"XLLM_SP_EXPRESS": "0"}),
    ("memo_4", {"XLLM_SP_MEMO_SLOTS": "4"}),          # nearly every insert fails
    ("memo_off", {"XLLM_SP_MEMO_SLOTS": "0"}),
    ("wide", {"XLLM_SP_FORCE_WIDE": "1"}),
    ("warm", {"XLLM_SP_WARM": "1"}),                  # BPE only: the warm-up pre-passes
]


@pytest.fixture(scope="module")
def gold():
    with open(GOLD) as f:
        return json.load(f)["models"]


@pytest.fixture(scope="module")
def dirs(tmp_path_factory, gold):
    """Model directories: the committed ones, and chain_unigram rebuilt from sp_unigram_4k (the bytes upstream ran
    on, by their SHA-256)."""
    root = tmp_path_factory.mktemp("sp_layouts")
    out = {n: ML.materialise(n, root) for n in ML.NAMES}
    for n, d in out.items():
        with open(os.path.join(d, "tokenizer.model"), "rb") as f:
            assert hashlib.sha256(f.read()).hexdigest() == gold[n]["sha256"], n
    return out


@pytest.fixture(scope="module")
def orcs(oracle, dirs):
    return {n: oracle.SentencePieceOracle(dirs[n]) for n in ML.NAMES}


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


def _longest_word(norm, split_mode):
    """Bytes of the longest word of a normalised text: a word starts at each U+2581 (split_mode 1), or at each U+2581
    that does not follow another one (split_mode 2)."""
    starts = [0]
    i = norm.find(SP, 1)
    while i >= 0:
        if split_mode == 1 or norm[i - 3:i] != SP:
            starts.append(i)
        i = norm.find(SP, i + 1)
    starts.append(len(norm))
    return max(b - a for a, b in zip(starts, starts[1:]))


def _want(orc, name, text, ids=None):
    """(ids, status) the device must produce: the oracle's ids, or XLLM_ERR_CAPACITY for a Unigram word past 511
    bytes."""
    if name in UNIGRAM and _longest_word(orc.normalize(text), ML.LAYOUT[name]["split_mode"]) > UNI_MAX_WORD:
        return [], ERR_CAPACITY
    return (orc.encode(text).tolist() if ids is None else ids), 0


def _encode(h, texts, stride):
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    return h.encode_batch(b.text, b.offsets, stride)


def _check(h, texts, want, stride=None):
    """ids, n_ids and status of every row: want[i] = (ids, status).  A row the stride truncates holds the expected
    prefix, with the full count and status 1; a refused row has n_ids 0 and its error status."""
    if stride is None:
        stride = max(16, max((len(w) for w, _ in want), default=0) + 8)
    ids, n_ids, status = _encode(h, texts, stride)
    bad = []
    for i, (w, st) in enumerate(want):
        if st < 0:
            ok = int(status[i]) == st and int(n_ids[i]) == 0
        else:
            keep = min(len(w), stride)
            ok = (int(n_ids[i]) == len(w) and int(status[i]) == (1 if len(w) > stride else 0)
                  and ids[i, :keep].tolist() == w[:keep])
        if not ok:
            bad.append((i, texts[i][:48], int(n_ids[i]), len(w), int(status[i]), st))
    assert not bad, (len(bad), bad[:4])
    return ids, n_ids, status


def _fuzz(name, seed, n=200):
    """Whitespace-heavy random texts (or chain texts for chain_unigram), checked against the oracle live."""
    rnd = random.Random(seed)
    if name == "chain_unigram":
        return ML.chain_texts(rnd)
    alphabet = ["a", "b", "cd", "efg", "word", " ", " ", "  ", "    ", "        ", "\t", "\n", "\r\n", "\x00", "▁",
                "é", "日本", "\U0001F600", "7", "42", "ﬁ", "\n    ", "\n        "]
    out = []
    for _ in range(n):
        out.append("".join(rnd.choice(alphabet) for _ in range(rnd.randrange(0, 160))).encode())
    for k in (7, 41, 170, 171, 300):
        out.append((" " * k).encode())
        out.append(("if x:\n" + " " * k + "return y\n").encode())
    return out


def _golden_batch(orcs, gold, name):
    """The goldens, then the generator's long seam texts and a fuzz set, both against the oracle."""
    cases = gold[name]["cases"]
    texts = [bytes.fromhex(c["text"]) for c in cases]
    want = [_want(orcs[name], name, t, c["ids"]) for t, c in zip(texts, cases)]
    more = ML.seam_texts(name) + _fuzz(name, 5)
    return texts + more, want + [_want(orcs[name], name, t) for t in more]


# ---------------------------------------------------------------------------- every model, every kernel variant
_CASES = [(n, v, e) for n in ML.NAMES for v, e in VARIANTS if not (v == "warm" and n in UNIGRAM)]


@pytest.mark.parametrize("name,variant,env", _CASES, ids=["%s-%s" % (n, v) for n, v, _ in _CASES])
def test_goldens_under_variants(dirs, orcs, gold, name, variant, env):
    texts, want = _golden_batch(orcs, gold, name)
    h = _handle(dirs[name], env)
    try:
        for _ in range(2):                      # a second launch on the same handle
            _check(h, texts, want)
    finally:
        h.close()
    if name == "ws_unigram":
        assert sum(st == ERR_CAPACITY for _, st in want) >= 10


@pytest.mark.parametrize("name", ML.NAMES)
def test_memo_carried_over_launches(dirs, orcs, gold, name):
    """xllm_set_memo_policy(N): words that hold U+2581 runs (and every other word) come out of a table filled by
    earlier launches."""
    texts, want = _golden_batch(orcs, gold, name)
    h = _handle(dirs[name])
    try:
        h.set_memo_policy(100000)
        for seed in (0, 1, 0, 2, 1):
            fz = _fuzz(name, 100 + seed, 120)
            _check(h, fz, [_want(orcs[name], name, t) for t in fz])
            _check(h, texts, want)
    finally:
        h.close()


# ---------------------------------------------------------------------------- strides that truncate
def test_truncate_inside_space_run_words(dirs, orcs):
    """llama_bpe / ws_unigram: rows cut at every id, so inside each word led by a U+2581 run and between the byte
    pieces of LF / tab / NUL."""
    for name in ("llama_bpe", "ws_unigram"):
        orc = orcs[name]
        texts = [b"def f(x):\n    if x:\n        return  x\n" * 3, b"a" + b" " * 37 + b"b\tc\r\n  d" + b" " * 9 + b"e",
                 b"   lead  and  trail   ", b"\n\n        x\x00\x00  y" * 4]
        want = [_want(orc, name, t) for t in texts]
        h = _handle(dirs[name])
        try:
            for stride in range(1, max(len(w) for w, _ in want) + 1):
                _check(h, texts, want, stride=stride)
        finally:
            h.close()


def test_truncate_after_express_handover(dirs, orcs):
    """nodummy_bpe: a non-ASCII char mid-prompt hands the request from the express kernel to the buffer path; the row
    is cut right before, at and after the first id the buffer path writes."""
    orc = orcs["nodummy_bpe"]
    rnd = random.Random(9)
    heads = [ML.words_text(rnd, n) for n in (60, 500, 520, 1030, 1600)]
    texts, cuts = [], set()
    for head in heads:
        for tail in (" été x y", "日本 word", "\U0001F600", " ①②"):
            t = (head + tail + " " + ML.words_text(rnd, 200)).encode()
            texts.append(t)
            n_head = len(orc.encode(head.encode()))
            cuts.update((n_head - 1, n_head, n_head + 1, n_head + 2))
    want = [_want(orc, "nodummy_bpe", t) for t in texts]
    h = _handle(dirs["nodummy_bpe"])
    try:
        for stride in sorted(cuts):
            _check(h, texts, want, stride=stride)
    finally:
        h.close()


def test_truncate_inside_long_word_pass(dirs, orcs):
    """nosplit_bpe: a prompt is one pre-token, so a long prompt's ids come from the long-word kernel; cut them at
    several points, with short neighbours that fit."""
    orc = orcs["nosplit_bpe"]
    from xllm_service_b200 import workload
    texts = [" ".join(workload.sentences(n // 60, (8, 12), seed=n)).encode()[:n] for n in (700, 1500, 3000, 6000)]
    texts += [b"of the", b"", b"a b c"]
    want = [_want(orc, "nosplit_bpe", t) for t in texts]
    h = _handle(dirs["nosplit_bpe"])
    try:
        for stride in (1, 3, 64, 200, 201, 511, 512, 513, 1000):
            _check(h, texts, want, stride=stride)
    finally:
        h.close()


# ---------------------------------------------------------------------------- Unigram words past the lattice
def test_unigram_word_too_long_is_refused(dirs, orcs):
    orc = orcs["ws_unigram"]
    texts = [b"hello world", b" " * 171, b"x" + b" " * 170 + b"y", b"x" + b" " * 171 + b"y", b"two words",
             b" " * 600 + b"a", b"a" * 600, b"a" + b" " * 175, b"indent\n" + b" " * 180 + b"x\nok", b" " * 169,
             b" " * 170]
    want = [_want(orc, "ws_unigram", t) for t in texts]
    # 170 U+2581 and "y": 511 bytes, the longest word that fits; the dummy prefix adds one U+2581 to a leading run
    assert [st for _, st in want] == [0, -6, 0, -6, 0, -6, -6, -6, -6, 0, -6]
    h = _handle(dirs["ws_unigram"])
    try:
        _check(h, texts, want)
    finally:
        h.close()


# ---------------------------------------------------------------------------- long-word scratch contention
def test_nosplit_many_long_requests(dirs, orcs):
    """More long requests than long-word scratch slots in one batch: 200 prompts of 1-3 KB and a few of 10-20 KB, each
    one pre-token."""
    from xllm_service_b200 import workload
    orc = orcs["nosplit_bpe"]
    rnd = random.Random(13)
    corpus = " ".join(workload.sentences(4000, (8, 12), seed=3)).encode()
    texts = []
    for i in range(204):
        n = rnd.randint(10000, 20000) if i % 50 == 7 else rnd.randint(1000, 3000)
        s = rnd.randrange(0, len(corpus) - n)
        texts.append(corpus[s:s + n])
    want = [_want(orc, "nosplit_bpe", t) for t in texts]
    for variant, env in (VARIANTS[0], VARIANTS[4]):
        h = _handle(dirs["nosplit_bpe"], env)
        try:
            _check(h, texts, want)
        finally:
            h.close()


# ---------------------------------------------------------------------------- end to end
def test_ingest_end_to_end_llama(oracle, dirs, orcs, gold):
    """One xllm_ingest_batch on llama_bpe in small pipeline chunks: ids, keys (the chained block hash of the ids) and
    the 16-bit id download."""
    from xllm_service_b200 import workload
    orc = orcs["llama_bpe"]
    texts = [bytes.fromhex(c["text"]) for c in gold["llama_bpe"]["cases"]] + _fuzz("llama_bpe", 77)
    b = workload.pack_prompts(texts)
    T = 1024
    h = _handle(dirs["llama_bpe"])
    try:
        h.set_pipeline(29, 1 << 14)
        out = h.ingest_batch(b.text, b.offsets, T, want_match=False)
        narrow = h.ingest_batch(b.text, b.offsets, T, want_match=False, ids_u16=True)
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
        n_blocks += keys.shape[0]
    assert n_blocks >= 20
    for f in ("n_ids", "status", "keys"):
        assert (narrow[f] == out[f]).all(), f
    for r in range(len(texts)):                 # a row's ids past its count are not part of the result
        n = min(int(out["n_ids"][r]), T)
        assert (narrow["ids"][r, :n].astype(np.int32) == out["ids"][r, :n]).all(), r
