#!/usr/bin/env python3
"""Goldens for the exact NFC check of tokenizers with `normalizer: NFC` (csrc/hf_nfc.cu, xllm_set_nfc_policy), minted
through the unchanged tests/golden/hf_qwen2_style/tokenizer.json with upstream HF `tokenizers` (pip 0.22.2):

  nfc      texts in NFC whose chars are not all NFC-inert (combining marks in a dozen scripts, seeded consonant + sign
           streams, marks next to an added token) -> ids (add_special_tokens = 1, as fast_tokenizer.cpp:20-30 calls it)
  not_nfc  texts NFC changes -> the wheel's NFC of them (recorded to show that it changes)
  wheel_older  texts Python's unicodedata (15.0) composes but the wheel's older Unicode data leaves alone: the device
           refuses them, the safe direction

Output (committed): tests/golden/hf_nfc_goldens.json
"""
import json
import os
import random
import unicodedata

HERE = os.path.dirname(os.path.abspath(__file__))
MODEL = os.path.join(HERE, "hf_qwen2_style", "tokenizer.json")
OUT = os.path.join(HERE, "hf_nfc_goldens.json")

SENTENCES = [
    "ภาษาไทยเป็นภาษาที่มีวรรณยุกต์ ผู้คนพูดกันทั่วประเทศ และเด็ก ๆ เรียนหนังสือที่โรงเรียน",        # Thai
    "ज़िंदगी एक सफ़र है, और हम सब मुसाफ़िर हैं। क़लम और काग़ज़ लेकर आओ।",                       # Devanagari, nukta
    "আমি বাংলায় গান গাই। আকাশে মেঘ করেছে, বাতাস বইছে।",                                      # Bengali
    "தமிழ் மொழி மிகவும் பழமையானது. நான் பாடம் படிக்கிறேன், அவள் கோயிலுக்குப் போனாள்.",       # Tamil
    "മലയാളം ഒരു ദ്രാവിഡ ഭാഷയാണ്. ഞാൻ ഇന്ന് പുസ്തകം വായിച്ചു, കൊച്ചി മനോഹരമാണ്.",           # Malayalam
    "ಕನ್ನಡ ಭಾಷೆ ತುಂಬಾ ಸುಂದರವಾಗಿದೆ. ನಾನು ಕೂಡ ಬರುತ್ತೇನೆ, ಕೋಟೆ ದೊಡ್ಡದು.",                    # Kannada
    "සිංහල භාෂාව ලස්සනයි. මම පොත කියවමි, ලෝකය විශාලයි.",                                    # Sinhala
    "မြန်မာဘာသာစကားသည် လှပသည်။ ကျွန်တော် စာဖတ်နေသည်။",                                      # Myanmar
    "ភាសាខ្មែរគឺជាភាសាផ្លូវការនៃប្រទេសកម្ពុជា។ ខ្ញុំចូលចិត្តអានសៀវភៅ។",                               # Khmer
    "بِسْمِ ٱللَّهِ ٱلرَّحْمَٰنِ ٱلرَّحِيمِ. اَلْعَرَبِيَّةُ لُغَةٌ جَمِيلَةٌ.",                     # Arabic, harakat
    "בְּרֵאשִׁית בָּרָא אֱלֹהִים אֵת הַשָּׁמַיִם וְאֵת הָאָרֶץ.",                                  # Hebrew, niqqud
    "Ἐν ἀρχῇ ἦν ὁ λόγος, καὶ ὁ λόγος ἦν πρὸς τὸν θεόν. ᾠδὴ καὶ ῥήτωρ.",                     # polytonic Greek
    "Tiếng Việt rất đẹp; café, naïve, Ångström, 한국어 문장, 日本語のかな、ガギグ。",            # precomposed, mixed
]
# consonant ranges and the signs that follow them, per script (seeded streams of consonant + sign)
STREAMS = [
    ((0x0E01, 0x0E2E), [0x0E31, 0x0E34, 0x0E35, 0x0E36, 0x0E37, 0x0E38, 0x0E39, 0x0E48, 0x0E49, 0x0E4A, 0x0E4B]),
    ((0x0915, 0x0939), [0x093C, 0x093E, 0x093F, 0x0940, 0x0941, 0x0942, 0x0947, 0x0948, 0x094B, 0x094D, 0x0902]),
    ((0x0995, 0x09A8), [0x09BC, 0x09BE, 0x09BF, 0x09C0, 0x09C1, 0x09C7, 0x09CB, 0x09CD, 0x09D7, 0x0981]),
    ((0x0B95, 0x0BA9), [0x0BBE, 0x0BBF, 0x0BC0, 0x0BC6, 0x0BC7, 0x0BCA, 0x0BCD, 0x0BD7]),
    ((0x0D15, 0x0D28), [0x0D3E, 0x0D3F, 0x0D46, 0x0D47, 0x0D4A, 0x0D4D, 0x0D57]),
    ((0x0C95, 0x0CA8), [0x0CBE, 0x0CBF, 0x0CC2, 0x0CC6, 0x0CCA, 0x0CCD, 0x0CD5, 0x0CD6]),
    ((0x0D9A, 0x0DA5), [0x0DCA, 0x0DCF, 0x0DD9, 0x0DDA, 0x0DDC, 0x0DDF]),
    ((0x1000, 0x1020), [0x102B, 0x102D, 0x102E, 0x102F, 0x1031, 0x1036, 0x1037, 0x1039, 0x103A]),
    ((0x0628, 0x0647), [0x064B, 0x064E, 0x064F, 0x0650, 0x0651, 0x0652, 0x0670]),
    ((0x05D0, 0x05EA), [0x05B0, 0x05B4, 0x05B7, 0x05B8, 0x05BC, 0x05C1, 0x05C2]),
]
NOT_NFC = [
    unicodedata.normalize("NFD", "Ti\u1ebfng Vi\u1ec7t r\u1ea5t \u0111\u1eb9p"),   # NFD Vietnamese
    "cafe\u0301", "\u212b angstrom sign", "\uf900 compatibility ideograph", "\u0958 excluded nukta form",
    "\u1100\u1161 Hangul L+V", "\uac00\u11a8 Hangul LV+T", "\u09c7\u09be Bengali o", "\u0bc6\u0bbe Tamil o",
    "\u304b\u3099 kana voicing", "a\u0301\u0316 ccc inversion", "\u0344 excluded non-starter decomposition",
]
WHEEL_OLDER = ["\U00011935\U00011930", "x \U00011935\U00011930 y"]   # Dives Akuru (Unicode 13): Python composes U+11938


def stream(rnd, cons, signs, n):
    out = []
    for _ in range(n):
        out.append(chr(rnd.randint(*cons)))
        for _ in range(rnd.choice((0, 1, 1, 2))):
            out.append(chr(rnd.choice(signs)))
        if rnd.random() < 0.15:
            out.append(" ")
    return "".join(out)


def nfc_texts():
    rnd = random.Random(15)
    texts = [unicodedata.normalize("NFC", s) for s in SENTENCES]
    for cons, signs in STREAMS:
        for n in (5, 40, 300):
            texts.append(unicodedata.normalize("NFC", stream(rnd, cons, signs, n)))
    texts += ["\u0915\u093c<|endoftext|>\u093f", "<|endoftext|>\u0301", "\u0995<|endoftext|>\u09be\u0995\u09be",
              "\u00e8<|endoftext|>\u0316", "\u0e01\u0e34<|endoftext|>\u0e48"]
    texts = [unicodedata.normalize("NFC", t) for t in texts]
    for t in texts:
        assert unicodedata.is_normalized("NFC", t), t
    return texts


def cases():
    from tokenizers import Tokenizer, normalizers
    tok = Tokenizer.from_file(MODEL)
    nfc = normalizers.NFC()
    out = {"nfc": [{"text": t.encode().hex(), "ids": tok.encode(t, add_special_tokens=True).ids} for t in nfc_texts()],
           "not_nfc": [], "wheel_older": []}
    for t in NOT_NFC:
        n = nfc.normalize_str(t)
        assert n != t, t
        out["not_nfc"].append({"text": t.encode().hex(), "wheel_nfc": n.encode().hex()})
    for t in WHEEL_OLDER:
        assert nfc.normalize_str(t) == t and unicodedata.normalize("NFC", t) != t, t
        out["wheel_older"].append({"text": t.encode().hex(), "python_nfc": unicodedata.normalize("NFC", t).encode().hex()})
    return out


def main():
    import tokenizers
    gold = cases()
    with open(OUT, "w") as f:
        json.dump({"tokenizers_version": tokenizers.__version__, "unidata_version": unicodedata.unidata_version,
                   "cases": gold}, f, separators=(",", ":"), ensure_ascii=True)
    print({k: len(v) for k, v in gold.items()})


if __name__ == "__main__":
    main()
