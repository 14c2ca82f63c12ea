"""The SentencePiece BPE kernels on models without byte fallback (tests/golden/make_sp_nobf_fixture.py), bit-exact
against the goldens upstream libsentencepiece produced and against the CPU oracle, through the C-ABI.  A char no piece
covers is <unk>, and a run of unknown symbols is one <unk>:

  nobf_bpe          split_mode 1 with the express kernel: a word with an unknown symbol is a hard word, merged by
                    express_long_word with the unknown flag carried in; a non-ASCII byte hands the request over
  nobf_ws_bpe       kept whitespace, U+2581-run words, tab / LF / CR unknown: the buffer path only
  nobf_nodummy_bpe  no dummy prefix: the first word of a request, or of a text piece, may start with an unknown
  nobf_nosplit_bpe  a whole text is one pre-token: unknown runs merged in the long-word pass (long_finish)

Each model runs under the kernel variants (express, memo size, wide ids, warm-up), with rows cut inside unknown runs,
a word memo carried across launches, pipelined ingest with block keys, and segmented requests.

In every layout the loader accepts, each word but a request's first starts with U+2581, a known piece (a suffix-space
model is refused, and a split_mode 0 request is one word).  So the unknown flag carried INTO a word (ExpReq::U across
express words, bit 2 of ExpResume, the drain's prev_unk at a word start) never meets an unknown first symbol, and no
text can tell it apart from false.  The merges inside a word (lane path, cooperative chunks, express_long_word,
long_finish) are what these texts pin."""
import hashlib
import importlib.util
import json
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
GOLD = os.path.join(HERE, "golden", "sp_nobf_goldens.json")


def _load_generator():
    spec = importlib.util.spec_from_file_location("make_sp_nobf_fixture",
                                                  os.path.join(HERE, "golden", "make_sp_nobf_fixture.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


MN = _load_generator()
EXPRESS = ("nobf_bpe", "nobf_nodummy_bpe")     # split_mode 1 + remove_extra_whitespaces: the express kernel runs

VARIANTS = [
    ("default", {}),                                  # express kernel (split_mode 1 models) + memo
    ("express_off", {"XLLM_SP_EXPRESS": "0"}),
    ("memo_4", {"XLLM_SP_MEMO_SLOTS": "4"}),          # nearly every insert fails
    ("memo_off", {"XLLM_SP_MEMO_SLOTS": "0"}),
    ("wide", {"XLLM_SP_FORCE_WIDE": "1"}),
    ("warm", {"XLLM_SP_WARM": "1"}),                  # the warm-up pre-passes
]


@pytest.fixture(scope="module")
def gold():
    with open(GOLD, encoding="utf-8") as f:
        return json.load(f)


@pytest.fixture(scope="module")
def dirs(tmp_path_factory, gold):
    """Model directories: the committed ones, and the nmt_nfkc ones with their charsmap put back (the bytes upstream
    ran on, by their SHA-256)."""
    root = tmp_path_factory.mktemp("sp_nobf")
    out = {n: MN.materialise(n, root) for n in MN.NAMES}
    for n, d in out.items():
        with open(os.path.join(d, "tokenizer.model"), "rb") as f:
            assert hashlib.sha256(f.read()).hexdigest() == gold["models"][n]["sha256"], n
    return out


@pytest.fixture(scope="module")
def orcs(oracle, dirs):
    return {n: oracle.SentencePieceOracle(dirs[n]) for n in MN.NAMES}


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


def _check(h, texts, want, stride=None):
    """ids, n_ids and status of every row against want[i]; a row the stride truncates holds the expected prefix, with
    the full count and status 1."""
    from xllm_service_b200 import workload
    if stride is None:
        stride = max(16, max((len(w) for w in want), default=0) + 8)
    b = workload.pack_prompts(texts)
    ids, n_ids, status = h.encode_batch(b.text, b.offsets, stride)
    bad = []
    for i, w in enumerate(want):
        keep = min(len(w), stride)
        if not (int(n_ids[i]) == len(w) and int(status[i]) == (1 if len(w) > stride else 0)
                and ids[i, :keep].tolist() == w[:keep]):
            bad.append((i, texts[i][:48], int(n_ids[i]), len(w), int(status[i])))
    assert not bad, (len(bad), bad[:4])


def _fuzz(seed, n=200):
    return MN.random_texts(random.Random(seed), n, 160)


def _golden_batch(orcs, gold, name):
    """The goldens, then the generator's long seam texts and a fuzz set, both against the oracle."""
    texts = [t.encode() for t in gold["texts"]]
    more = MN.seam_texts() + _fuzz(5)
    return texts + more, gold["models"][name]["ids"] + [orcs[name].encode(t).tolist() for t in more]


# ---------------------------------------------------------------------------- every model, every kernel variant
_CASES = [(n, v, e) for n in MN.NAMES for v, e in VARIANTS]


@pytest.mark.parametrize("name,variant,env", _CASES, ids=["%s-%s" % (n, v) for n, v, _ in _CASES])
def test_goldens_under_variants(dirs, orcs, gold, name, variant, env):
    texts, want = _golden_batch(orcs, gold, name)
    h = _handle(dirs[name], env)
    try:
        for _ in range(2):                      # a second launch on the same handle
            _check(h, texts, want)
    finally:
        h.close()


# ---------------------------------------------------------------------------- the express kernel's seams
def _unk_word(rnd, n, where):
    """A word of n bytes whose unknown run (1..3 symbols, at most n) is at its start, end or both."""
    k = min(n, rnd.randint(1, 3))
    if where == "start":
        return MN.unk_run(rnd, k) + MN.letters(rnd, n - k)
    if where == "end":
        return MN.letters(rnd, n - k) + MN.unk_run(rnd, k)
    if n < 2:
        return MN.unk_run(rnd, n)
    return MN.unk_run(rnd, 1) + MN.letters(rnd, n - 2) + MN.unk_run(rnd, 1)


def _short_words(rnd, n):
    return " ".join(MN.letters(rnd, rnd.randint(1, 3)) for _ in range(n))


def express_seam_texts():
    """Words that start or end with unknown symbols where an express step has its seams: ending on and starting at a
    512-byte window's last byte, as word 62..66 of a step (a step resolves 64), behind 0..15 bytes of alignment, in
    front of a hand-over, and as the 15 / 16 / 17-byte words between the lane path and express_long_word."""
    rnd = random.Random(64)
    t = []
    ends = ("start", "end", "both")
    for where in ends:
        for n in (1, 3, 8, 15, 16, 17, 40, 300):
            w = _unk_word(rnd, n, where)
            # the word's last byte at text offset 509 .. 1024, then its first byte at 511, 512, 1023
            for start in [last + 1 - n for last in (509, 510, 511, 512, 513, 1022, 1023, 1024)] + [511, 512, 1023]:
                pre = MN.words_text(rnd, start - 1).ljust(start - 1, "q") + " " if start > 0 else ""
                t.append(pre + w + " " + _unk_word(rnd, rnd.randint(1, 6), where) + " tail")
    for k in range(60, 68):                                           # the unknown word is word k of a step
        for where in ends:
            for n in (2, 5, 15, 16, 30):
                t.append(_short_words(rnd, k) + " " + _unk_word(rnd, n, where) + " " + _short_words(rnd, 70))
        t.append(_short_words(rnd, k) + " " + MN.unk_run(rnd, 40) + " " + _short_words(rnd, 70))
    for off in range(16):                                             # every start alignment
        for where in ends:
            for n in (1, 4, 15, 16, 17):
                w = _unk_word(rnd, n, where)
                t.append(" " * off + w + " " + w + " " + _short_words(rnd, 40))
                t.append(MN.letters(rnd, off + 1) + " " + w + " x")
    for sp in ("é", "日本", "\U0001F600", "ø", "\xa0", SPACE_MARK):   # directly before a hand-over
        for lead in (0, 1, 100, 505, 510, 511, 512, 1000):
            pre = MN.words_text(rnd, lead)
            for glue in ("", " ", "  "):
                for where in ends:
                    w = _unk_word(rnd, rnd.choice((1, 5, 15, 20)), where)
                    t.append(pre + (" " if pre else "") + w + glue + sp + glue + w + " more words after")
    for n in (16, 17, 100, 511, 512, 513, 600, 1100):                 # hard words too long for the lane path
        t.append("head " + MN.word_with_unknowns(rnd, n) + " " + MN.word_with_unknowns(rnd, n, min(n, 70)) + " end")
    return [s.encode() for s in t]


SPACE_MARK = "▁"


def test_express_seams(dirs, orcs):
    """nobf_bpe and nobf_nodummy_bpe: the express kernel and the buffer-path kernel alone (XLLM_SP_EXPRESS=0) both
    equal the oracle."""
    texts = express_seam_texts()
    for name in EXPRESS:
        want = [orcs[name].encode(t).tolist() for t in texts]
        assert sum(w.count(orcs[name].encode(b"|")[-1]) for w in want) > 1000
        for env in ({}, {"XLLM_SP_EXPRESS": "0"}):
            h = _handle(dirs[name], env)
            try:
                _check(h, texts, want)
            finally:
                h.close()


@pytest.mark.parametrize("name", MN.NAMES)
def test_express_kernel_runs_where_it_should(dirs, name):
    """The launch plan: the express kernel is one of the tokenizer kernels of every ingest_batch chunk for the
    split_mode 1 models (and not when switched off, or for the others), so the seams above run through it."""
    from xllm_service_b200 import workload
    texts = MN.random_texts(random.Random(3), 900, 60)
    b = workload.pack_prompts(texts)
    for env, express in (({}, name in EXPRESS), ({"XLLM_SP_EXPRESS": "0"}, False)):
        h = _handle(dirs[name], env)
        try:
            h.set_pipeline(200, 1 << 20)
            h.ingest_batch(b.text, b.offsets, 256, want_match=False)
            chunks, launches = h.last_batch_stats()
        finally:
            h.close()
        assert chunks > 1
        assert launches == ((3 if express else 2) + 2) * chunks, (env, chunks, launches)   # + row prep + hash


# ---------------------------------------------------------------------------- a memo that outlives its launch
@pytest.mark.parametrize("name", MN.NAMES)
def test_memo_carried_over_batches(dirs, orcs, gold, name):
    """xllm_set_memo_policy(N): words (with and without unknowns) filled in by one batch are looked up by the next,
    through encode_batch and through ingest_batch in several pipeline chunks."""
    from xllm_service_b200 import workload
    orc = orcs[name]
    rnd = random.Random(8)
    vocab = [MN.letters(rnd, rnd.randint(1, 8)) for _ in range(150)]
    vocab += [_unk_word(rnd, rnd.randint(1, 15), w) for w in ("start", "end", "both") for _ in range(50)]
    vocab += [MN.unk_run(rnd, k) for k in (1, 2, 3, 15)] + ["é" + MN.unk_run(rnd, 2)]

    def batch(seed):
        r = random.Random(seed)
        return [" ".join(r.choice(vocab) for _ in range(r.randint(1, 200))).encode() for _ in range(150)]

    h = _handle(dirs[name])
    try:
        h.set_memo_policy(100000)
        for seed in (0, 1, 0, 2, 1):
            texts = batch(seed)
            _check(h, texts, [orc.encode(t).tolist() for t in texts])
        h.set_pipeline(37, 1 << 14)
        for seed in (3, 0, 3):
            texts = batch(seed)
            b = workload.pack_prompts(texts)
            out = h.ingest_batch(b.text, b.offsets, 2048, want_match=False)
            for r, t in enumerate(texts):
                want = orc.encode(t).tolist()
                assert out["n_ids"][r] == len(want) and out["status"][r] == 0, (seed, r)
                assert out["ids"][r, :len(want)].tolist() == want, (seed, r)
    finally:
        h.close()


# ---------------------------------------------------------------------------- strides that cut unknown runs
def _cuts(orc, texts):
    """Strides that end a row right before, on and after each <unk> id."""
    unk = orc.encode(b"|")[-1]
    cuts = set()
    for t in texts:
        for i, x in enumerate(orc.encode(t).tolist()):
            if x == unk:
                cuts.update((i, i + 1, i + 2))
    return sorted(c for c in cuts if c > 0)


def test_truncate_inside_unknown_runs(dirs, orcs):
    """Rows cut at and around every <unk>: in the express kernel (nobf_bpe, both the lane path and express_long_word),
    in the buffer path (express off, and the kept-whitespace model), and in the long-word pass (a 1100-byte word, and
    the cross-word model's whole-text pre-token)."""
    rnd = random.Random(21)
    short = ["ab|| cd ~x y^ {a} " * 4, "x " + MN.word_with_unknowns(rnd, 15) + " " + MN.word_with_unknowns(rnd, 40),
             "w " + MN.word_with_unknowns(rnd, 300, 45) + " z"]
    long_ = ["s " + MN.word_with_unknowns(rnd, 1100) + " e", MN.word_with_unknowns(rnd, 700, 66)]
    plans = [("nobf_bpe", {}, short + long_), ("nobf_bpe", {"XLLM_SP_EXPRESS": "0"}, short),
             ("nobf_ws_bpe", {}, short + ["a\t|\n  |b " * 5]), ("nobf_nosplit_bpe", {}, long_ + [" ".join(short)])]
    for name, env, ts in plans:
        orc = orcs[name]
        texts = [t.encode() for t in ts]
        want = [orc.encode(t).tolist() for t in texts]
        h = _handle(dirs[name], env)
        try:
            for stride in _cuts(orc, texts):
                _check(h, texts, want, stride=stride)
        finally:
            h.close()


# ---------------------------------------------------------------------------- segmented requests
def test_segments_do_not_carry_the_unknown_flag(oracle, dirs, orcs):
    """nobf_nodummy_bpe: text pieces that end and start with unknowns, back to back in one request and split by id
    spans.  Each piece is its own encode call, so the <unk> that starts a piece stays even when the piece before ended
    with one."""
    from xllm_service_b200 import workload
    orc = orcs["nobf_nodummy_bpe"]
    rnd = random.Random(17)
    reqs = []
    for i in range(60):
        segs = []
        for j in range(rnd.randint(2, 6)):
            if j and rnd.random() < 0.25:
                segs.append(np.arange(rnd.randint(1, 9), dtype=np.int32) + 100)
            else:
                body = _short_words(rnd, rnd.choice((0, 1, 5, 80, 300)))
                segs.append((MN.unk_run(rnd, rnd.randint(1, 3)) + body + " " * (i % 2) + MN.unk_run(rnd, 2)).encode())
        reqs.append(segs)
    reqs += [[b"|", b"|", b"|"], [b"ab|", b"|cd"], [b"||", np.full(3, 7, np.int32), b"||"], [b"|" * 40, b"|" * 40]]
    pieces, seg_len, spans, rss, want = [], [], [], [0], []
    for segs in reqs:
        ids = []
        for s in segs:
            if isinstance(s, bytes):
                pieces.append(s)
                seg_len.append(-1)
                ids += orc.encode(s).tolist()
            else:
                spans.append(s)
                seg_len.append(s.size)
                ids += s.tolist()
        rss.append(len(seg_len))
        want.append(ids)
    unk = orc.encode(b"|")[-1]
    assert sum(w.count(unk) for w in want) >= 300
    pb = workload.pack_prompts(pieces)
    b = workload.SegmentBatch(pb.text, pb.offsets, np.asarray(rss, np.int32), np.asarray(seg_len, np.int32),
                              np.concatenate(spans).astype(np.int32), np.zeros(len(reqs), bool),
                              np.zeros(len(reqs), np.int32))
    T = 1024
    h = _handle(dirs["nobf_nodummy_bpe"])
    try:
        h.set_pipeline(13, 1 << 12)
        out = h.ingest_batch_segments(b, T, want_match=False)
    finally:
        h.close()
    for r, w in enumerate(want):
        assert out["status"][r] == 0 and out["n_ids"][r] == len(w), r
        assert out["ids"][r, :len(w)].tolist() == w, r
        keys = oracle.block_hash_chain(np.asarray(w, np.int32))
        assert (out["keys"][r, :keys.shape[0]] == keys).all(), r


# ---------------------------------------------------------------------------- end to end, with block keys
@pytest.mark.parametrize("name", MN.NAMES)
def test_ingest_block_keys(oracle, dirs, orcs, gold, name):
    """One pipelined xllm_ingest_batch per model: ids, and block keys equal to the chained block hash of the oracle's
    ids (truncated rows hash their first T ids)."""
    from xllm_service_b200 import workload
    orc = orcs[name]
    texts = [t.encode() for t in gold["texts"]] + MN.seam_texts() + _fuzz(77, 100)
    b = workload.pack_prompts(texts)
    T = 1024
    h = _handle(dirs[name])
    try:
        h.set_pipeline(29, 1 << 14)
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
        n_blocks += keys.shape[0]
    assert n_blocks >= 40
