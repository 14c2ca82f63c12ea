"""The exact NFC check of tokenizers with `normalizer: NFC` (csrc/hf_nfc.cu) without a GPU: its generated tables
(csrc/unicode_nfc.inc) against Python's unicodedata for every code point, the rule it implements (tests/nfc_oracle.py)
against unicodedata.is_normalized, the property the device relies on — every text it accepts is left unchanged by
the `tokenizers` wheel's NFC, whole and per segment between added tokens — and the committed goldens."""
import json
import os
import random
import re
import sys
import unicodedata

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import nfc_oracle  # noqa: E402

INC = os.path.join(os.path.dirname(HERE), "xllm_service_b200", "csrc", "unicode_nfc.inc")
ALPHABET = nfc_oracle.FUZZ_ALPHABET
CONTEXTS = [("", ""), ("a", ""), ("e", "́"), ("á", "̖"), ("a̖", "́"), ("ᄀ", "x")]


def _random_strings(n, seed):
    rnd = random.Random(seed)
    return ["".join(rnd.choice(ALPHABET) for _ in range(rnd.randrange(0, 14))) for _ in range(n)]


def _array(name, text):
    m = re.search(r"static const unsigned (?:short|int|long long) %s\[(\d+)\] = \{(.*?)\};" % name, text, re.S)
    vals = [int(v.rstrip("ul"), 0) for v in re.findall(r"0x[0-9A-Fa-f]+ull|0x[0-9A-Fa-f]+|\d+", m.group(2))]
    assert len(vals) == int(m.group(1)), name
    return vals


def test_tables_against_unicodedata():
    with open(INC) as f:
        text = f.read()
    assert "unicodedata %s" % unicodedata.unidata_version in text.splitlines()[0]
    s1, s2 = _array("kNfcStage1", text), _array("kNfcStage2", text)
    ccc, qc = nfc_oracle.props()
    for cp in range(0x110000):
        v = s2[s1[cp >> 8] * 256 + (cp & 255)]
        assert (v & 0xFF, v >> 8) == (ccc[cp], qc[cp]), hex(cp)
    assert sum(1 for q in qc if q == nfc_oracle.QC_NO) == 1120 and sum(1 for q in qc if q == nfc_oracle.QC_MAYBE) == 111
    keys, dec = _array("kNfcDecompCp", text), _array("kNfcDecomp", text)
    assert keys == sorted(keys) and len(keys) == 2061
    listed = dict(zip(keys, (dec[4 * i:4 * i + 4] for i in range(len(keys)))))
    for cp in range(0x110000):
        if 0xD800 <= cp < 0xE000 or 0xAC00 <= cp < 0xAC00 + 11172:
            continue
        nfd = [ord(c) for c in unicodedata.normalize("NFD", chr(cp))]
        got = [v for v in listed[cp] if v] if cp in listed else [cp]
        assert got == nfd, hex(cp)
    ck, cv = _array("kNfcCompKey", text), _array("kNfcComp", text)
    assert ck == sorted(ck) and len(ck) == len(cv) == 941
    for k, c in zip(ck, cv):
        a, b = k >> 21, k & 0x1FFFFF
        assert unicodedata.normalize("NFC", chr(a) + chr(b)) == chr(c)
        assert unicodedata.decomposition(chr(c)) == "%04X %04X" % (a, b)


def test_rule_matches_is_normalized_on_random_strings():
    """200 K strings: without the chunk cap the rule is exactly is_normalized; with it, accepted implies NFC."""
    for s in _random_strings(200_000, 1):
        b = s.encode()
        want = 0 if unicodedata.is_normalized("NFC", s) else 1
        assert nfc_oracle.nfc_verdict(b, cap=1 << 30) == want, [hex(ord(c)) for c in s]
        assert nfc_oracle.nfc_verdict(b) in (want, 1)


def test_rule_on_every_scalar_value_in_context():
    for pre, post in CONTEXTS:
        for cp in range(0x110000):
            if 0xD800 <= cp < 0xE000:
                continue
            s = pre + chr(cp) + post
            want = 0 if unicodedata.is_normalized("NFC", s) else 1
            assert nfc_oracle.nfc_verdict(s.encode(), cap=1 << 30) == want, (hex(cp), pre, post)


def test_cap_and_malformed():
    v = nfc_oracle.nfc_verdict
    assert v(("x" + "́" * 31).encode()) == 0 and v(("x" + "́" * 32).encode()) == 1   # 32 / 33 code points
    assert v(("a" + "̖" * 100).encode()) == 0          # no Maybe char: no cap
    for bad in (b"\xff", b"\xc0\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"a\xcc", b"e\xcc\x81\x80"):
        assert v(bad) == 2, bad
    assert v("é".encode() + b"\xff") == 2              # malformed wins over not NFC


def test_accepted_texts_are_fixed_points_of_the_wheels_nfc():
    """Every text the device accepts is left unchanged by the wheel's NFC — its Unicode data is older than Python's,
    so equality with Python's NFC alone would not be enough — and so is every segment between added tokens, which
    the crate normalises one at a time."""
    tokenizers = pytest.importorskip("tokenizers")
    nfc = tokenizers.normalizers.NFC()
    rnd = random.Random(2)
    accepted = []
    for s in _random_strings(200_000, 3):
        if rnd.random() < 0.5:
            k = rnd.randrange(0, len(s) + 1)
            s = s[:k] + "<|x|>" + s[k:]
        if nfc_oracle.nfc_verdict(s.encode()) == 0:
            accepted.append(s)
    for pre, post in CONTEXTS:
        for cp in range(0x110000):
            if not 0xD800 <= cp < 0xE000:
                s = pre + chr(cp) + post
                if nfc_oracle.nfc_verdict(s.encode()) == 0:
                    accepted.append(s)
    assert len(accepted) > 1_000_000
    pieces = [p for s in accepted for p in s.split("<|x|>")]
    # NFC never composes or reorders across U+000A, so one call checks a block of texts; a mismatch names the text
    for i in range(0, len(pieces), 20_000):
        block = pieces[i:i + 20_000]
        if nfc.normalize_str("\n".join(block)) != "\n".join(block):
            bad = [p for p in block if nfc.normalize_str(p) != p]
            assert not bad, [[hex(ord(c)) for c in p] for p in bad[:5]]
    for s in accepted[:200_000]:
        assert nfc.normalize_str(s) == s


def test_goldens_regenerate_against_the_wheel():
    pytest.importorskip("tokenizers")
    import make_hf_nfc_fixture as m
    with open(m.OUT) as f:
        gold = json.load(f)
    assert m.cases() == gold["cases"]
    for c in gold["cases"]["nfc"]:
        assert nfc_oracle.nfc_verdict(bytes.fromhex(c["text"])) == 0
    for c in gold["cases"]["not_nfc"] + gold["cases"]["wheel_older"]:
        assert nfc_oracle.nfc_verdict(bytes.fromhex(c["text"])) == 1
