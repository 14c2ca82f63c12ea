"""The HF `tokenizer.json` backend on added-token sets of real sizes and shapes (tests/golden/make_hf_added_fixture.py:
an adversarial GPT-2 set, Llama-3's 256, Qwen2's chat / FIM / tool tokens, DeepSeek-V3's ~800, 256 tokens past id
65 535): hf_mark_added's leftmost-longest passes (normalized:false tokens first, normalized:true ones between them),
the pre-tokenizer rules around added tokens, the staging-buffer seams, the word-list cap, the other entry points and
the legacy C ABI, bit for bit against the goldens from pip `tokenizers` and the CPU oracle."""
import ctypes
import functools
import os
import random
import re
import sys
import unicodedata

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
import make_hf_added_fixture as fx  # noqa: E402
from test_gpu_memo import VARIANTS, _handle  # noqa: E402
from test_oracle_hf_added import GOLD, _limit_set, limit_sets  # noqa: E402


def _kNBuf():
    with open(os.path.join(HERE, "..", "xllm_service_b200", "csrc", "sp_encode.cu")) as f:
        return int(re.search(r"constexpr int kNBuf = (\d+);", f.read()).group(1))


SEAM = _kNBuf()


@pytest.fixture(scope="module")
def derived(tmp_path_factory):
    d = tmp_path_factory.mktemp("hf_added")
    return {name: fx.write(name, str(d)) for name in fx.SETS}


@functools.lru_cache(maxsize=None)
def _oracle(path):
    from oracle import oracle as o
    o.build()
    return o.HfBpeOracle(path)


def _want(h, texts):
    return [h.prefix_ids + h.encode(t).tolist() + h.suffix_ids for t in texts]


def _encode_all(tok, texts, stride=None):
    from xllm_service_b200 import workload
    b = workload.pack_prompts(texts)
    stride = stride or max(16, 3 * max((len(t) for t in texts), default=0) + 8)
    ids, n_ids, status = tok.encode_batch(b.text, b.offsets, stride)
    return [ids[i, :n_ids[i]].tolist() for i in range(len(texts))], status


def _check(tok, texts, want):
    got, status = _encode_all(tok, texts, max(16, max(len(w) for w in want) + 8))
    bad = [(i, t[:60], g[:8], w[:8]) for i, (t, g, w, s) in enumerate(zip(texts, got, want, status)) if s != 0 or g != w]
    assert not bad, (len(bad), bad[:3])


def _set_texts(name):
    """Every token's contexts and random strings, as bytes (for the NFC model, those in NFC)."""
    rnd = random.Random(fx.hash_seed(name) + 11)
    return [s.encode() for s in fx.texts(name, rnd, 400)
            if name != "qwen2_chat" or unicodedata.is_normalized("NFC", s)]


def _env(name, env):
    """The NFC model runs under the exact NFC check: a text in NFC with combining marks is encoded, not refused."""
    return dict(env, XLLM_HF_NFC_VERIFY="1") if name == "qwen2_chat" else env


@pytest.mark.parametrize("vname,env", VARIANTS)
@pytest.mark.parametrize("name", fx.SETS)
def test_goldens_and_oracle(derived, name, vname, env):
    g = GOLD["sets"][name]
    h = _oracle(derived[name])
    # the library normalizes text that is not in NFC; the device refuses it (-5) and never rewrites a text
    refused = [s.encode() for s, _ in g["cases"] if name == "qwen2_chat" and not unicodedata.is_normalized("NFC", s)]
    cases = [(s.encode(), ids) for s, ids in g["cases"] if s.encode() not in refused]
    tok = _handle(derived[name], _env(name, env))
    try:
        assert tok.vocab_size() == g["vocab_size"]
        _check(tok, [s for s, _ in cases], [ids for _, ids in cases])
        if refused:
            assert (_encode_all(tok, refused)[1] == -5).all()
        texts = _set_texts(name)
        _check(tok, texts, _want(h, texts))
    finally:
        tok.close()


def _seam_texts(name):
    """The set's longest token slid over every offset around the first staging seam, after fillers that end in the
    places the pre-tokenizer looks back at; and the long second-pass token of gpt2_adv against the 64-byte token."""
    toks = [c for c, _, _, _ in fx.TOKENS[name]()]
    longest = max(toks, key=lambda c: len(c.encode()))
    L = len(longest.encode())
    out = []
    for lead in ("ab ", "x  ", "é' ", "12 ", "日本 ", "a\n\n"):   # short pre-tokens: a run of 2 KB would be too long
        filler = (lead * (SEAM // len(lead.encode()) + 2)).encode()
        for start in range(SEAM - L - 16, SEAM + 9):
            head = filler[:start].decode("utf-8", "ignore").encode()      # whole chars only
            head = head + b"z" * (start - len(head))
            out.append(head + longest.encode() + b"'ll  y " + toks[1].encode() + b" tail")
    for k in (4, 8):    # a whitespace run right before the token: one pre-token only when the token is seen as one
        for start in range(SEAM - L - 16, SEAM + 9):
            head = (b"ab " * (start // 3 + 1))[:start - k - 1] + b"b" + b" " * k
            out.append(head + longest.encode() + b" tail")
    # the second and third seams: those buffers begin at the tail the previous one left (about L + 8 bytes short of
    # the seam each), so the window widens by that much per buffer
    for k in (2, 3):
        for start in range(k * SEAM - (k - 1) * (L + 24) - L - 16, k * SEAM + 9):
            head = (b"ab " * (start // 3 + 1))[:start]
            out.append(head + longest.encode() + b"'ll  y " + toks[1].encode() + b" tail")
            head = (b"ab " * (start // 3 + 1))[:start - 5] + b"b" + b" " * 4
            out.append(head + longest.encode() + b" tail")
    if name == "gpt2_adv":
        for start in list(range(SEAM - 100, SEAM + 9)) + list(range(2 * SEAM - 200, 2 * SEAM + 9)):
            out.append((b"q " * start)[:start] + b"z" * 12 + fx.LONG64.encode() + b" end")
            out.append(b"q " * (start // 2) + b"z" * 12 + b"<|long" + b" end")
    return out


@pytest.mark.parametrize("name", fx.SETS)
def test_long_texts_and_seams(derived, name):
    h = _oracle(derived[name])
    toks = [c for c, _, _, _ in fx.TOKENS[name]()]
    rnd = random.Random(5)
    texts = _seam_texts(name)
    texts.append(("~<a>" * 5000).encode() if name == "gpt2_adv" else "".join(toks[:8] * 400).encode())   # word list cap
    texts.append("".join("x %s " % rnd.choice(toks) for _ in range(3000)).encode())
    texts.append("".join(rnd.choice(toks) + rnd.choice(["日本語", "カタカナ", " 中文", "123", "\n"]) for _ in range(2500)).encode())
    texts.append(" ".join(rnd.choice(toks + ["word", "日本", "don't"]) for _ in range(9000))[:20000].encode())
    for vname, env in (VARIANTS[0], VARIANTS[2], VARIANTS[3]):
        tok = _handle(derived[name], _env(name, env))
        try:
            _check(tok, texts, _want(h, texts))
        finally:
            tok.close()


@pytest.mark.parametrize("verify", [False, True])
def test_qwen2_chat_nfc_policies(derived, verify):
    """Combining marks next to the chat tokens: under the exact check a text in NFC is encoded and one that is not is
    refused (-5); under the default inert-char proof an accepted text is right and an ASCII one is accepted."""
    h = _oracle(derived["qwen2_chat"])
    toks = [c for c, _, _, _ in fx.TOKENS["qwen2_chat"]()]
    rnd = random.Random(9)
    marks = ["́", "̈", "̣́", "̸", "é", "가", "x́́"]
    texts = []
    for t in toks:
        for m in marks:
            texts += [t + m + "y", "a" + m + t, m + t + m, t + m + t]
    texts += ["".join(rnd.choice(toks + marks + ["a", " ", "é", "日"]) for _ in range(20)) for _ in range(300)]
    tok = _handle(derived["qwen2_chat"], {})
    try:
        if verify:
            tok.set_nfc_policy(1)
        got, status = _encode_all(tok, [t.encode() for t in texts])
    finally:
        tok.close()
    for t, g, s in zip(texts, got, status):
        nfc = unicodedata.is_normalized("NFC", t)
        if verify:
            assert s == (0 if nfc else -5), repr(t)
        elif t.isascii():
            assert s == 0, repr(t)
        if s == 0:
            assert g == _want(h, [t.encode()])[0], repr(t)


def test_other_entry_points(derived):
    """ingest_batch with block keys, ingest_batch_segments, and rows the stride truncates inside and right after an
    added token: ids equal the oracle's, a truncated row holds the oracle's prefix with the full count and status 1."""
    from oracle import oracle as o
    from xllm_service_b200 import workload
    import xllm_service_b200 as x
    import numpy as np
    for name in ("gpt2_adv", "wide_256"):
        h = _oracle(derived[name])
        texts = _set_texts(name)[:600]
        want = _want(h, texts)
        tok = x.Ingest(tokenizer_path=derived[name])
        try:
            b = workload.pack_prompts(texts)
            T = (max(len(w) for w in want) // tok.block_size + 2) * tok.block_size
            res = tok.ingest_batch(b.text, b.offsets, T, want_keys=True, want_match=False)
            for i, w in enumerate(want):
                assert res["status"][i] == 0 and res["ids"][i, :len(w)].tolist() == w, (name, i)
                keys = o.block_hash_chain(np.array(w, dtype=np.int32))
                assert (res["keys"][i, :keys.shape[0]] == keys).all(), (name, i)
            # segments: text pieces encoded on their own and appended, with an id span between
            pieces = [t for t in texts[:200]]
            rss, seg_len, span, ptexts = [0], [], [], []
            for r in range(100):
                seg_len += [-1, 3, -1]
                span += [7, 8, 9]
                ptexts += [pieces[2 * r], pieces[2 * r + 1]]
                rss.append(len(seg_len))
            pb = workload.pack_prompts(ptexts)
            sb = workload.SegmentBatch(pb.text, pb.offsets, np.array(rss, np.int32), np.array(seg_len, np.int32),
                                       np.array(span, np.int32), np.zeros(100, bool), np.zeros(100, np.int32))
            out = tok.ingest_batch_segments(sb, T, want_keys=False, want_match=False)
            for r in range(100):
                w = (h.prefix_ids + h.encode(pieces[2 * r]).tolist() + h.suffix_ids + [7, 8, 9] +
                     h.prefix_ids + h.encode(pieces[2 * r + 1]).tolist() + h.suffix_ids)
                assert out["status"][r] == 0 and out["ids"][r, :out["n_ids"][r]].tolist() == w, (name, r)
            # truncation inside / right after an added token
            tk = max((c for c, _, _, _ in fx.TOKENS[name]()), key=len)
            t = ("word " * 20 + tk + tk + " tail").encode()
            w = _want(h, [t])[0]
            k = w.index(h.token_to_id(tk))
            for stride in (k, k + 1, k + 2):
                b2 = workload.pack_prompts([t])
                ids, n_ids, status = tok.encode_batch(b2.text, b2.offsets, stride)
                assert status[0] == 1 and n_ids[0] == len(w) and ids[0, :stride].tolist() == w[:stride], stride
        finally:
            tok.close()


def _legacy():
    import xllm_service_b200 as x
    L = ctypes.CDLL(x.lib_path())
    L.tokenizers_new_from_path.restype = ctypes.c_void_p
    L.tokenizers_new_from_path.argtypes = [ctypes.c_char_p]
    L.tokenizers_decode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int,
                                    ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_size_t)]
    L.tokenizers_id_to_token.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.POINTER(ctypes.c_char_p),
                                         ctypes.POINTER(ctypes.c_size_t)]
    L.tokenizers_token_to_id.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_int32)]
    L.tokenizers_get_vocab_size.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]
    L.tokenizers_free.argtypes = [ctypes.c_void_p]
    return L


@pytest.mark.parametrize("name", fx.SETS)
def test_legacy_abi(derived, name):
    """tokenizers_decode with skip 0 / 1 (non-special added tokens kept, every token through the ByteLevel decoder,
    lossy UTF-8), tokenizers_id_to_token / token_to_id for every added token, tokenizers_get_vocab_size."""
    g = GOLD["sets"][name]
    L = _legacy()
    hd = L.tokenizers_new_from_path(os.path.join(derived[name], "tokenizer.json").encode())
    assert hd
    try:
        data, m = ctypes.c_char_p(), ctypes.c_size_t()
        for ids, plain, skipped in g["decode"]:
            arr = (ctypes.c_uint32 * len(ids))(*ids)
            for skip, want in ((0, plain), (1, skipped)):
                L.tokenizers_decode(hd, arr, len(ids), skip, ctypes.byref(data), ctypes.byref(m))
                assert ctypes.string_at(data, m.value).decode("utf-8") == want, (ids, skip)
        out = ctypes.c_int32()
        for (c, _, _, _), i in zip(fx.TOKENS[name](), g["token_ids"]):
            L.tokenizers_token_to_id(hd, c.encode(), len(c.encode()), ctypes.byref(out))
            assert out.value == i, c
            L.tokenizers_id_to_token(hd, i, ctypes.byref(data), ctypes.byref(m))
            assert ctypes.string_at(data, m.value) == c.encode(), c
        n = ctypes.c_size_t()
        L.tokenizers_get_vocab_size(hd, ctypes.byref(n))
        assert n.value == g["vocab_size"]
    finally:
        L.tokenizers_free(hd)


def test_largest_accepted_set_runs(tmp_path):
    """2048 tokens in exactly 65 535 bytes load on the device and encode as the oracle does."""
    import xllm_service_b200 as x
    name, contents, ok = limit_sets()[0]
    assert ok and len(contents) == 2048
    path = _limit_set(tmp_path, name, contents)
    h = _oracle(path)
    rnd = random.Random(2)
    texts = [" ".join(rnd.choice(contents + ["<t1", "x", "word"]) for _ in range(rnd.randrange(1, 30))).encode()
             for _ in range(300)]
    tok = x.Ingest(tokenizer_path=path)
    try:
        _check(tok, texts, _want(h, texts))
    finally:
        tok.close()
