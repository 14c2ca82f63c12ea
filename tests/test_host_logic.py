"""Host-side logic of the product that needs no GPU: the SentencePiece model loader's table building
(csrc/sp_model.cc, through xllm_tokenizer_probe), error codes, and the workload generator."""
import os

import numpy as np
import pytest

HERE = os.path.dirname(__file__)
MODEL_DIR = os.path.join(HERE, "golden", "sp_bpe_8k")


@pytest.fixture(scope="module", autouse=True)
def built():
    import __graft_entry__ as ge
    ge.build()


def test_tokenizer_probe_fixture():
    from xllm_service_b200 import _lib
    info = _lib.tokenizer_probe(MODEL_DIR)
    assert info["n_pieces"] == 8000 and info["byte_fallback"] == 1 and info["unk_id"] == 0
    assert info["split_mode"] == 1          # no piece holds U+2581 past its first char: words split exactly
    assert info["n_symbols"] >= info["n_pieces"]
    assert info["n_pairs"] > 8000 and info["n_pair_slots"] >= 4 * info["n_pairs"]   # load factor <= 0.25
    assert info["trie_units"] > 0 and 3 <= info["max_unit_out"] <= 64
    # the file form and the directory form resolve to the same model
    assert _lib.tokenizer_probe(os.path.join(MODEL_DIR, "tokenizer.model")) == info


def test_tokenizer_probe_errors(tmp_path):
    import xllm_service_b200 as x
    from xllm_service_b200 import _lib
    with pytest.raises(x.IngestError) as e:
        _lib.tokenizer_probe(str(tmp_path / "nope"))
    assert e.value.code == -3  # XLLM_ERR_IO
    (tmp_path / "tokenizer.model").write_bytes(b"not a protobuf \xff\xff\xff")
    with pytest.raises(x.IngestError) as e:
        _lib.tokenizer_probe(str(tmp_path))
    assert e.value.code in (-4, -5)


def test_unigram_models_load_and_odd_ones_are_rejected(tmp_path):
    """Unigram models load (Viterbi tables); a model whose pieces span word starts has no exact word split and is
    refused, as are WORD / CHAR models — never mis-tokenised."""
    spm = pytest.importorskip("sentencepiece")
    import io
    import xllm_service_b200 as x
    from xllm_service_b200 import _lib, workload
    info = _lib.tokenizer_probe(os.path.join(HERE, "golden", "sp_unigram_4k"))
    assert info["n_pieces"] == 4000 and info["split_mode"] == 1 and info["n_pairs"] == 0
    for name, kw in (("cross", dict(model_type="unigram", split_by_whitespace=False)), ("word", dict(model_type="word")),
                     ("char", dict(model_type="char"))):
        model = io.BytesIO()
        spm.SentencePieceTrainer.train(sentence_iterator=iter(workload.sentences(6000, seed=1)), model_writer=model,
                                       vocab_size={"cross": 4000, "word": 300, "char": 30}[name], minloglevel=2, **kw)
        d = tmp_path / name
        d.mkdir()
        (d / "tokenizer.model").write_bytes(model.getvalue())
        with pytest.raises(x.IngestError) as e:
            _lib.tokenizer_probe(str(d))
        assert e.value.code == -5, name  # XLLM_ERR_UNSUPPORTED


def test_workload_exact_tokens_and_shared_prefixes(oracle):
    from xllm_service_b200 import workload
    sp = oracle.SentencePieceOracle(MODEL_DIR)
    vocab = workload.make_vocabulary()
    assert len(vocab) == 20000 and len(set(vocab)) == 20000 and all(2 <= len(w) <= 9 for w in vocab)
    wb = workload.pack_prompts(vocab)
    _, wcnt = sp.encode_batch(wb.text, wb.offsets, 32, n_threads=4)
    T = 512
    b, meta = workload.make_prompts_exact_tokens(
        200, T, wcnt, seed=3, shared_prefix=dict(n_prefixes=6, frac=0.8, min_blocks=1, max_blocks=3, block_tokens=128))
    b2, _ = workload.make_prompts_exact_tokens(
        200, T, wcnt, seed=3, shared_prefix=dict(n_prefixes=6, frac=0.8, min_blocks=1, max_blocks=3, block_tokens=128))
    assert (b.text == b2.text).all() and (b.offsets == b2.offsets).all()   # deterministic
    ids, n = sp.encode_batch(b.text, b.offsets, T + 8, n_threads=4)
    assert (n == T).all()
    pid = meta["prefix_id"]
    assert 0.6 < (pid >= 0).mean() < 0.95
    for j in np.unique(pid[pid >= 0]):
        rows = np.nonzero(pid == j)[0]
        L = int(meta["prefix_blocks"][rows[0]]) * 128
        assert (ids[rows, :L] == ids[rows[0], :L]).all()


def test_factory_selects_tiktoken_by_tokenizer_class(tmp_path):
    """TokenizerFactory::create_tokenizer (tokenizer_factory.cpp:9-32): tokenizer_class == TikTokenTokenizer
    -> tiktoken tables (bytes are symbols, no pre-split, no normaliser); otherwise SentencePiece."""
    import shutil
    from xllm_service_b200 import _lib
    info = _lib.tokenizer_probe(os.path.join(HERE, "golden", "tiktoken_1k"))
    assert info["split_mode"] == 0 and info["trie_units"] == 0 and info["byte_fallback"] == 0
    assert info["n_pieces"] == 1453            # 256 bytes + 1200 merges - 3 bytes dropped on purpose
    assert info["n_symbols"] == 1456           # the 3 rank-less bytes are still symbols (they emit nothing)
    assert info["n_pairs"] >= 1200
    # only the TOP-LEVEL key counts (tokenizer_args.cpp:49-51 reads "tokenizer_class" from the root object): a nested
    # one — here inside auto_map, placed first in the file — must not select the tiktoken backend
    d2 = tmp_path / "nested"
    d2.mkdir()
    shutil.copy(os.path.join(HERE, "golden", "tiktoken_1k", "tokenizer.model"), d2 / "tokenizer.model")
    (d2 / "tokenizer_config.json").write_text(
        '{"auto_map": {"tokenizer_class": "TikTokenTokenizer"}, "tokenizer_class": "LlamaTokenizer"}')
    with pytest.raises(_lib.IngestError):
        _lib.tokenizer_probe(str(d2))          # falls through to SentencePiece, which cannot read a tiktoken file
    d3 = tmp_path / "toplevel_last"
    d3.mkdir()
    shutil.copy(os.path.join(HERE, "golden", "tiktoken_1k", "tokenizer.model"), d3 / "tokenizer.model")
    (d3 / "tokenizer_config.json").write_text(
        '{"auto_map": {"tokenizer_class": "Other"}, "x": [1, {"tokenizer_class": "Nope"}], '
        '"tokenizer_class": "TikTokenTokenizer"}')
    assert _lib.tokenizer_probe(str(d3))["n_pieces"] == info["n_pieces"]
    # the same vocabulary file without the tokenizer_class hint is NOT silently read as tiktoken
    d = tmp_path / "plain"
    d.mkdir()
    shutil.copy(os.path.join(HERE, "golden", "tiktoken_1k", "tokenizer.model"), d / "tokenizer.model")
    import xllm_service_b200 as x
    with pytest.raises(x.IngestError):
        _lib.tokenizer_probe(str(d))


HF_DIR = os.path.join(HERE, "golden", "hf_bpe_8k")


def test_hf_tokenizer_json_tables(tmp_path):
    """tokenizer.json wins the factory's choice (tokenizer_factory.cpp:14-19) and loads as byte-level BPE."""
    import json
    import shutil
    import xllm_service_b200 as x
    from xllm_service_b200 import _lib
    info = _lib.tokenizer_probe(HF_DIR)
    assert info["split_mode"] == 3 and info["trie_units"] == 0 and info["byte_fallback"] == 0
    assert info["n_pieces"] == 8000 and info["n_symbols"] == 8000
    assert info["n_pairs"] == 8000 - 256 - 1          # one merge per non-byte, non-special token
    assert _lib.tokenizer_probe(os.path.join(HF_DIR, "tokenizer.json")) == info
    # a directory holding BOTH files is an HF tokenizer, as in the reference's factory
    both = tmp_path / "both"
    both.mkdir()
    shutil.copy(os.path.join(HF_DIR, "tokenizer.json"), both / "tokenizer.json")
    shutil.copy(os.path.join(MODEL_DIR, "tokenizer.model"), both / "tokenizer.model")
    assert _lib.tokenizer_probe(str(both))["split_mode"] == 3
    # configurations the device path does not implement are refused, never approximated
    with open(os.path.join(HF_DIR, "tokenizer.json")) as f:
        base = json.load(f)

    def variant(name, edit):
        d = json.loads(json.dumps(base))
        edit(d)
        q = tmp_path / name
        q.mkdir()
        (q / "tokenizer.json").write_text(json.dumps(d))
        return str(q)

    def set_(path, value):
        def f(d):
            for k in path[:-1]:
                d = d[k]
            d[path[-1]] = value
        return f

    def pre_of(style):
        with open(os.path.join(HERE, "golden", style, "tokenizer.json")) as f:
            return json.load(f)["pre_tokenizer"]

    def sequence(pre, edit):   # another fixture's pre_tokenizer Sequence, its entries edited
        def f(d):
            d["pre_tokenizer"] = json.loads(json.dumps(pre))
            edit(d["pre_tokenizer"]["pretokenizers"])
        return f

    cl100k, deepseek = pre_of("hf_llama3_style"), pre_of("hf_deepseek_style")
    for name, edit in (
        ("nfkc", set_(["normalizer"], {"type": "NFKC"})),
        ("other_regex", set_(["pre_tokenizer"], {"type": "Sequence", "pretokenizers": [
            {"type": "Split", "pattern": {"Regex": "\\p{N}{1,3}"}, "behavior": "Isolated", "invert": False},
            {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": True, "use_regex": False}]})),
        ("dropout", set_(["model", "dropout"], 0.1)),
        ("prefix_space", set_(["pre_tokenizer", "add_prefix_space"], True)),
        ("no_regex", set_(["pre_tokenizer", "use_regex"], False)),
        ("whitespace", set_(["pre_tokenizer"], {"type": "Whitespace"})),
        ("cl100k_merged", sequence(cl100k, lambda s: s[0].__setitem__("behavior", "MergedWithPrevious"))),
        ("cl100k_invert", sequence(cl100k, lambda s: s[0].__setitem__("invert", True))),
        ("cl100k_byte_level_regex", sequence(cl100k, lambda s: s[1].__setitem__("use_regex", True))),
        ("deepseek_order", sequence(deepseek, lambda s: s.insert(0, s.pop(1)))),
        ("deepseek_no_byte_level", sequence(deepseek, lambda s: s.pop())),
        ("byte_level_alone", sequence(cl100k, lambda s: s.pop(0))),
        ("wordpiece", set_(["model", "type"], "WordPiece")),
        ("truncation", set_(["truncation"], {"max_length": 8, "strategy": "LongestFirst", "stride": 0, "direction": "Right"})),
        ("lstrip", lambda d: d["added_tokens"][0].__setitem__("lstrip", True)),
        ("roberta", set_(["post_processor"], {"type": "RobertaProcessing", "sep": ["</s>", 2], "cls": ["<s>", 0],
                                               "trim_offsets": True, "add_prefix_space": True})),
    ):
        with pytest.raises(x.IngestError) as e:
            _lib.tokenizer_probe(variant(name, edit))
        assert e.value.code == -5, name
    (tmp_path / "broken").mkdir()
    (tmp_path / "broken" / "tokenizer.json").write_text('{"model": {"vocab": {"a": 0}, "merges": [')
    with pytest.raises(x.IngestError) as e:
        _lib.tokenizer_probe(str(tmp_path / "broken"))
    assert e.value.code == -4
    # NFC (checked per request on device) and ignore_merges are accepted; so are the Llama-3 / Qwen2 layouts
    assert _lib.tokenizer_probe(variant("nfc", set_(["normalizer"], {"type": "NFC"})))["split_mode"] == 3
    assert _lib.tokenizer_probe(variant("im", set_(["model", "ignore_merges"], True)))["split_mode"] == 3
    for style in ("hf_llama3_style", "hf_qwen2_style"):
        assert _lib.tokenizer_probe(os.path.join(HERE, "golden", style))["split_mode"] == 3
    # ... and the refused sequences above are refused for their edit alone
    for name, pre in (("cl100k", cl100k), ("deepseek", deepseek)):
        assert _lib.tokenizer_probe(variant(name, sequence(pre, lambda s: None)))["split_mode"] == 3
    # a template post-processor is accepted (ids are wrapped on device)
    tp = {"type": "TemplateProcessing",
          "single": [{"SpecialToken": {"id": "<|endoftext|>", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}}],
          "pair": [{"Sequence": {"id": "A", "type_id": 0}}, {"Sequence": {"id": "B", "type_id": 1}}],
          "special_tokens": {"<|endoftext|>": {"id": "<|endoftext|>", "ids": [0], "tokens": ["<|endoftext|>"]}}}
    assert _lib.tokenizer_probe(variant("template", set_(["post_processor"], tp)))["split_mode"] == 3


def test_pipeline_chunk_schedule(tmp_path):
    """csrc/pipeline_schedule.h: every (batch size, chunk bound) is covered exactly by chunks in [1, bound] —
    including the 513..1536-request batches a first version of the tail rule turned into empty chunks."""
    import subprocess
    exe = tmp_path / "pipeline_schedule_main"
    subprocess.check_call(["g++", "-std=c++17", "-O2", os.path.join(HERE, "cpp", "pipeline_schedule_main.cc"), "-o", str(exe)])
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout[-1500:]


def test_micro_batcher_threading_against_a_stub(tmp_path):
    """host/ingest_batcher.h without a GPU: the three C-ABI entry points it calls are stubbed (a prompt "tokenises" to
    its bytes); three thread / batch-size / wait-window mixes (32 x 300 requests into batches of 64, 100 threads into
    batches of 16, 48 threads with no wait window): every caller gets its own prompt back, requests are coalesced
    into near-full batches while the device is busy, two device calls never overlap, and an oversized prompt is
    refused rather than queued forever.  (Also run under -fsanitize=thread when the batcher changes.)"""
    import subprocess
    exe = tmp_path / "batcher_stub_main"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-pthread", "-I", os.path.join(os.path.dirname(HERE), "include"),
                           "-I", os.path.join(os.path.dirname(HERE), "xllm_service_b200", "host"),
                           os.path.join(HERE, "cpp", "batcher_stub_main.cc"), "-o", str(exe)])
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout[-1000:]
