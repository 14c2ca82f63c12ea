"""Reference statement of the device's exact NFC check (xllm_service_b200/csrc/hf_nfc.cu) in Python, from
`unicodedata` alone: it never reads the generated tables (csrc/unicode_nfc.inc), so the tests that compare the two
check the tables against an independent source.

  boundary char = canonical combining class (ccc) 0 and NFC_Quick_Check Yes;
  chunk = a boundary char, or the start of the text, followed by the maximal run of non-boundary chars.
  A text is in NFC iff (1) no char has NFC_QC = No, (2) no two adjacent chars a, b have ccc(a) > ccc(b) > 0,
  (3) every chunk that holds an NFC_QC = Maybe char is left unchanged by NFC.
The device refuses a Maybe chunk longer than `cap` code points even when it is in NFC."""
import unicodedata

QC_YES, QC_MAYBE, QC_NO = 0, 1, 2
# combining-heavy alphabet for fuzzing: starters that compose, marks of many classes, Maybe chars, Hangul jamo and
# syllables, excluded and singleton decompositions, Indic two-part vowels, Dives Akuru
FUZZ_ALPHABET = ("aeoAEuiknsyzAO \n<>|" + "\u0300\u0301\u0302\u0303\u0308\u030a\u030c\u0327\u0328\u0316\u0323\u0331"
                 "\u093c\u094d\u05b0\u05b4\u05bc\u05c1\u064e\u0651\u0670\u0655\u0340\u0344\u0341\u0654\u0345"
                 "\u0915\u0928\u0930\u0933\u09be\u09cc\u09bc\u0b3e\u0b48\u0b57\u0bbe\u0bc6\u0bc7\u0bd7\u0cbf"
                 "\u0cc2\u0cc6\u0cd5\u0cd6\u0d3e\u0d4c\u0dca\u0dcf\u0dde\u0e38\u0e48\u1026\u1100\ud558\u1175"
                 "\u11a8\u11c2\uac00\uac01\u3099\u309a\u304b\u212b\uf900\u0958\u1e0a\u0387\u1f00\u0391\u0399"
                 "\U00011935\U00011930\U0001d165\U0001d16d\u0f71\u0f72\u0f80\u0e01\u00e9\u00c5")
_PROPS = None


def props():
    """bytearray pair (ccc, NFC_Quick_Check) indexed by code point.  NFC_QC as UAX #15 derives it: No = NFC changes the
    char on its own; Maybe = the char is the second half of a primary composite (Hangul V and T jamo included)."""
    global _PROPS
    if _PROPS is None:
        ccc, qc = bytearray(0x110000), bytearray(0x110000)
        second = set(range(0x1161, 0x1176)) | set(range(0x11A8, 0x11C3))
        for cp in range(0x110000):
            if 0xD800 <= cp < 0xE000:
                continue
            ch = chr(cp)
            ccc[cp] = unicodedata.combining(ch)
            if unicodedata.normalize("NFC", ch) != ch:
                qc[cp] = QC_NO
            d = unicodedata.decomposition(ch)
            if d and not d.startswith("<"):
                parts = d.split()
                if len(parts) == 2:
                    a, b = chr(int(parts[0], 16)), chr(int(parts[1], 16))
                    if unicodedata.normalize("NFC", a + b) == ch:
                        second.add(ord(b))
        for cp in second:
            if qc[cp] == QC_YES:
                qc[cp] = QC_MAYBE
        _PROPS = (ccc, qc)
    return _PROPS


def nfc_verdict(text: bytes, cap=32):
    """0: in NFC (the device tokenises it); 1: not in NFC, or a Maybe chunk longer than `cap` code points; 2: not valid
    UTF-8 (strict: no surrogates, overlong forms or code points past U+10FFFF)."""
    try:
        s = text.decode("utf-8")
    except UnicodeDecodeError:
        return 2
    ccc, qc = props()
    prev = 0
    start, has_maybe = 0, False
    for i, ch in enumerate(s):
        cp = ord(ch)
        c, q = ccc[cp], qc[cp]
        if q == QC_NO or (prev > c > 0):
            return 1
        prev = c
        if c == 0 and q == QC_YES:      # a boundary char closes the chunk before it
            if has_maybe and not _chunk_ok(s[start:i], cap):
                return 1
            start, has_maybe = i, False
        has_maybe |= q == QC_MAYBE
    if has_maybe and not _chunk_ok(s[start:], cap):
        return 1
    return 0


def _chunk_ok(chunk, cap):
    return len(chunk) <= cap and unicodedata.normalize("NFC", chunk) == chunk
