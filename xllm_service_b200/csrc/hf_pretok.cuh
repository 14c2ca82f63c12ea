// hf_pretok.cuh — warp-parallel pre-tokenizer of the HF byte-level BPE backend (included by sp_encode.cu).
//
// Device replacement for the two steps the Rust crate runs before BPE inside tokenizers_encode
// (xllm_service/tokenizer/tokenizers/src/lib.rs:83-99 -> Tokenizer::encode):
//   added_vocabulary.rs   split the text on the added tokens, leftmost-longest, verbatim: the normalized:false ones,
//                         then the normalized:true ones between those
//   pre_tokenizers/       split every remaining segment with the model's pattern, T.hf_pattern:
//   1  GPT-2 ByteLevel (oracle/hf_bpe_oracle.cc gpt2_split)
//        's|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+
//   2  the cl100k-family Split regex of the newer layouts, Llama-3: K = 3, Qwen2: K = 1 (oracle: cl100k_split)
//        (?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,K}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
//   3  DeepSeek-V3 / R1: Sequence[Split(\p{N}{1,3}), Split([一-龥぀-ゟ゠-ヿ]+), Split(main regex)], all Isolated —
//      numbers (groups of 3) and CJK / kana runs are cut out first and bound everything else; inside the remaining
//      pieces (oracle: ds3_split)
//        [!-/:-@\[-`{-~][A-Za-z]+|[^\r\n\p{L}\p{P}\p{S}]?[\p{L}\p{M}]+| ?[\p{P}\p{S}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
//
// The leftmost-first regex scan is sequential as written, but every token boundary of these patterns is decided by a
// window of one char back, one char ahead (plus two ASCII bytes after an apostrophe) and a few facts that need a scan
// along the buffer, done 32 bytes at a time with a warp-uniform carry.  So the warp decides all positions of the
// staging buffer at once, in passes (hf_scan):
//   A       hf_classify            class of every char (Unicode tables), UTF-8 validation, NFC quick check
//   A2      hf_mark_added          added-token starts, leftmost-longest, non-overlapping (one or two passes)
//   B1      hf_mark_contractions   contraction starts (patterns 1, 2)
//   C1, C2  hf_run_facts           swallowed CR/LFs, digit index in its run, CR/LF ahead in a whitespace run (2, 3)
//   D1, D2  hf_ascii_runs          "punct + ASCII letters" tokens (3)
//   B2      hf_token_start         token starts: the rules every pattern shares, then hf_rules1 / 2 / 3
// hf_rulesN is the device form of rulesN in tests/test_hf_rules_equivalence.py, which checks each rule set against
// the sequential scan.
#pragma once

// Per-byte scratch of hf_scan: two bytes per text byte, cls[] in the merge scratch S[] and aux[] in PM[], both idle
// while scanning.  Bit, pass that writes it, patterns that read it:
// cls[]
//   0x80       kHfCont        A    UTF-8 continuation byte (the whole byte)                                   all
//   bits 0-1   class          A    letter / number / whitespace / other; pattern 3: \p{M} is a letter, CJK   all
//                                  and kana are other
//   0x04       kHfIsSp        A    the char is U+0020                                                         all
//   0x08       kHfInAdded     A2   inside an added token, not its first byte (the whole byte)                 all
//   0x10       kHfAddedStart  A2   an added token starts here (the whole byte)                                all
//   0x20/0x40  kHfContr2/3    B1   a contraction of 2 / 3 bytes starts here                                   1, 2
// aux[] (patterns 2 and 3 only)
//   0x01  kAuxNl          A    CR or LF                                                                  2, 3
//   0x02  kAuxSwallowed   C1   a CR/LF that only CR/LFs separate from a punctuation char                2, 3
//   0x04  kAuxDigitStart  C1   a digit whose index in its run is a multiple of K                        2, 3
//   0x08  kAuxNlAfter     C2   whitespace other than CR/LF with a CR/LF later in its run                2, 3
//   0x10  kAuxPS          A    \p{P} or \p{S}                                                           3
//   0x20  kAuxCjk         A    char of the CJK / kana ranges (the whole byte)                           3
//   0x40  kAuxAStart      D1   ASCII punctuation that opens a "punct + ASCII letters" token             3
//   0x80  kAuxAIn         D2   ASCII letter inside such a token                                         3
enum : uint8_t { kHfOther = 0, kHfLetter = 1, kHfNumber = 2, kHfSpace = 3 };
constexpr uint8_t kHfIsSp = 0x04, kHfInAdded = 0x08, kHfAddedStart = 0x10, kHfContr2 = 0x20, kHfContr3 = 0x40,
                  kHfContr = 0x60, kHfCont = 0x80;
constexpr uint8_t kAuxNl = 0x01, kAuxSwallowed = 0x02, kAuxDigitStart = 0x04, kAuxNlAfter = 0x08;
constexpr uint8_t kAuxPS = 0x10, kAuxCjk = 0x20, kAuxAStart = 0x40, kAuxAIn = 0x80;
constexpr uint16_t kHfSpecialWord = 0x8000;  // wstart[] flag: the word is an added token (one id, no BPE)
constexpr uint16_t kHfPosMask = 0x0FFF;
__device__ __forceinline__ bool hf_ascii_alpha(uint8_t b) { return (uint8_t)((b | 0x20) - 'a') < 26; }
__device__ __forceinline__ bool hf_ascii_punct(uint8_t b) {
  return (b >= 0x21 && b <= 0x2F) || (b >= 0x3A && b <= 0x40) || (b >= 0x5B && b <= 0x60) || (b >= 0x7B && b <= 0x7E);
}
__device__ __forceinline__ bool hf_cjk(uint32_t cp) {   // [一-龥぀-ゟ゠-ヿ]
  return (cp >= 0x4E00 && cp <= 0x9FA5) || (cp >= 0x3040 && cp <= 0x30FF);
}

// class in bits 0-1; bit 2 (non-ASCII only): the char is not NFC-inert (scripts/gen_unicode_classes.py)
constexpr uint8_t kUniNfcSuspect = 0x04;
__device__ __forceinline__ uint8_t hf_class(const SpDev& T, uint32_t cp) {
  if (cp < 0x80) {
    const uint32_t l = cp | 0x20;
    if (l >= 'a' && l <= 'z') return kHfLetter;
    if (cp >= '0' && cp <= '9') return kHfNumber;
    if (cp == ' ' || (cp >= 9 && cp <= 13)) return kHfSpace;
    return kHfOther;
  }
  return __ldg(T.uni2 + (uint32_t)__ldg(T.uni1 + (cp >> 8)) * 256u + (cp & 255u));
}

// longest added token of added[a0, a1) that is a prefix of p[0..avail); 0 = none.  *id = its token id.
__device__ __forceinline__ int hf_added_len(const SpDev& T, const uint8_t* p, int avail, int32_t* id, uint32_t a0,
                                            uint32_t a1) {
  int best = 0;
  for (uint32_t a = a0; a < a1; ++a) {
    const int o = __ldg(T.added_off + a), l = (int)__ldg(T.added_off + a + 1) - o;
    if (l > avail || l <= best) continue;
    bool eq = true;
    for (int k = 0; k < l && eq; ++k) eq = p[k] == __ldg(T.added_blob + o + k);
    if (eq) { best = l; *id = __ldg(T.added_id + a); }
  }
  return best;
}

// ignore_merges: raw bytes of a pre-token -> id of the vocabulary entry with exactly those bytes, or -1.
// Table entry (16 B): x,y = FNV-1a 64 of the bytes (0 = empty), z = id, w = blob offset << 10 | length.
__device__ __forceinline__ int32_t hf_vocab_lookup(const SpDev& T, const uint8_t* w, int n) {
  if (n > 1023) return -1;
  unsigned long long h = 0xcbf29ce484222325ull;
  for (int k = 0; k < n; ++k) h = (h ^ w[k]) * 0x100000001b3ull;
  if (h == 0) h = 1;
  // FNV's upper bits barely move for 1-2 byte keys: mix before taking the slot (same on the host, hf_model.cc)
  uint32_t slot = (uint32_t)(((h ^ (h >> 29)) * 0xBF58476D1CE4E5B9ull) >> 32) & T.vtab_mask;
  for (;;) {
    const uint4 e = __ldg(T.vtab + slot);
    if ((e.x | e.y) == 0) return -1;
    if (e.x == (uint32_t)h && e.y == (uint32_t)(h >> 32) && (int)(e.w & 1023u) == n) {
      const uint8_t* b = T.vblob + (e.w >> 10);
      uint32_t diff = 0;  // no early exit: the loads are independent and overlap
      for (int k = 0; k < n; ++k) diff |= (uint32_t)(__ldg(b + k) ^ w[k]);
      if (diff == 0) return (int32_t)e.z;
    }
    slot = (slot + 1) & T.vtab_mask;
  }
}

struct HfScan {
  int nwords;      // complete pre-tokens listed in wstart[0..nwords); wstart[nwords] = tail_start
  int tail_start;  // first byte that is not part of a listed pre-token
  bool capped;     // wstart[] filled up: scan the kept tail again
  int bad;         // 0 ok, 1 malformed UTF-8, 2 the text is not provably in NFC and the tokenizer normalises with NFC
};

// ---- idioms of the passes below
__device__ __forceinline__ bool hf_added(uint8_t c) { return (c & (kHfInAdded | kHfAddedStart)) != 0; }
// start of the char that holds byte q (q itself unless it is a continuation byte)
__device__ __forceinline__ int hf_char_start(const uint8_t* cls, int q) {
  while (q > 0 && cls[q] == kHfCont) --q;
  return q;
}
// byte length of the char whose first byte is b0
__device__ __forceinline__ int hf_char_len(uint8_t b0) { return b0 < 0xC0 ? 1 : (b0 < 0xE0 ? 2 : (b0 < 0xF0 ? 3 : 4)); }
// forward scans: the bit of `bits` at the highest lane of `sel` (masked to the lanes below this one: the nearest such
// lane below), or `carry` from the previous 32 bytes when `sel` is empty
__device__ __forceinline__ bool hf_last_bit(uint32_t sel, uint32_t bits, bool carry) {
  return sel ? ((bits >> (31 - __clz(sel))) & 1u) != 0 : carry;
}
// forward scans: how many bits of `bits` lie above the highest lane of `sel`, or `carry` + all of them when `sel` is empty
__device__ __forceinline__ int hf_count_after(uint32_t sel, uint32_t bits, int carry) {
  return sel ? __popc(bits & ~((2u << (31 - __clz(sel))) - 1u)) : carry + __popc(bits);
}

// ---- A: classes + UTF-8 validation (+ the NFC quick check: every char NFC-inert => NFC is the identity).
// Returns HfScan::bad.
__device__ __forceinline__ int hf_classify(const SpDev& T, const uint8_t* nb, uint8_t* cls, uint8_t* aux, int nlen,
                                           bool final, int pattern, int lane) {
  const bool p3 = pattern == 3, with_aux = pattern == 2 || pattern == 3;
  bool bad = false, nfc_bad = false;
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    if (p < nlen) {
      const uint8_t b0 = nb[p];
      uint8_t v;
      uint8_t ax = (b0 == '\n' || b0 == '\r') ? kAuxNl : 0;
      if (b0 < 0x80) {
        v = hf_class(T, b0) | (b0 == ' ' ? kHfIsSp : 0);
        if (p3 && hf_ascii_punct(b0)) ax |= kAuxPS;
      } else if ((b0 & 0xC0) == 0x80) {
        v = kHfCont;
        bool cov = false;  // must belong to a lead byte at most 3 back
        for (int k = 1; k <= 3 && p - k >= 0; ++k) {
          const uint8_t x = nb[p - k];
          if ((x & 0xC0) == 0x80) continue;
          cov = hf_char_len(x) > k;
          break;
        }
        bad |= !cov;
      } else {
        const int l = hf_char_len(b0);
        v = kHfOther;
        if (p + l > nlen) {
          bad |= final;  // cut by the end of the text; otherwise the rest arrives with the next window
        } else {
          bool valid;
          utf8_unit(nb + p, (uint32_t)(nlen - p), b0, &valid);
          if (!valid) bad = true;
          else {
            const uint32_t cp = l == 2 ? (((b0 & 0x1Fu) << 6) | (nb[p + 1] & 0x3Fu))
                              : l == 3 ? (((b0 & 0x0Fu) << 12) | ((nb[p + 1] & 0x3Fu) << 6) | (nb[p + 2] & 0x3Fu))
                                       : (((b0 & 0x07u) << 18) | ((nb[p + 1] & 0x3Fu) << 12) | ((nb[p + 2] & 0x3Fu) << 6) | (nb[p + 3] & 0x3Fu));
            const uint8_t tb = hf_class(T, cp);   // bits 0-1 class, 2 NFC-suspect, 3-4: 1 P, 2 S, 3 M (class 0 only)
            nfc_bad |= T.nfc_check && !T.nfc_verdict && (tb & kUniNfcSuspect);   // verified: hf_nfc.cu
            v = tb & 3;
            if (p3) {
              const uint8_t sub = (tb >> 3) & 3;
              if (hf_cjk(cp)) { v = kHfOther; ax = kAuxCjk; }
              else if (v == kHfOther && sub == 3) v = kHfLetter;          // \p{M} runs with the letters
              else if (v == kHfOther && sub != 0) ax |= kAuxPS;
            }
          }
        }
      }
      cls[p] = v;
      if (with_aux) aux[p] = ax;
    }
  }
  __syncwarp();
  return __any_sync(kFull, bad) ? 1 : (__any_sync(kFull, nfc_bad) ? 2 : 0);
}

// ---- A2: added tokens, leftmost-longest, non-overlapping, over added[0, n).  n = n_added, or in the two-pass kernels
// n_added_plain: the normalized:false tokens, and hf_mark_added_second matches the normalized:true ones between them.
__device__ __forceinline__ void hf_mark_added(const SpDev& T, const uint8_t* nb, uint8_t* cls, int nlen, uint32_t n,
                                              int lane) {
  int cover = 0;
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    int al = 0;
    if (p < nlen) {
      const uint8_t b0 = nb[p];
      if ((T.added_first[b0 >> 5] >> (b0 & 31)) & 1u) {
        int32_t id;
        al = hf_added_len(T, nb + p, nlen - p, &id, 0, n);
      }
    }
    uint32_t m = __ballot_sync(kFull, al > 0);
    while (m) {
      const int bit = __ffs(m) - 1;
      m &= m - 1;
      const int q = base + bit;
      const int l = __shfl_sync(kFull, al, bit);
      if (q >= cover) {
        for (int k = lane; k < l; k += 32) cls[q + k] = k == 0 ? kHfAddedStart : kHfInAdded;
        cover = q + l;
      }
    }
  }
  __syncwarp();
}

// The second pass: a normalized token matches only between the tokens of the first pass (avail ends at the next
// one).  In a non-final buffer a first-pass token that the buffer end cuts off is not seen, so a match that reaches
// the last added_max_len bytes is deferred: the returned bound (nlen when nothing is deferred) lies 9 bytes below its
// start, the margin of the first pass, and the next buffer decides it.  Only the two-pass kernels (MODE 3) have it.
__device__ __forceinline__ int hf_mark_added_second(const SpDev& T, const uint8_t* nb, uint8_t* cls, int nlen, bool final,
                                                 int lane) {
  int cover = 0, bound = nlen;
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    int al = 0;
    if (p < nlen && !hf_added(cls[p])) {
      const uint8_t b0 = nb[p];
      if ((T.added_first[b0 >> 5] >> (b0 & 31)) & 1u) {
        int avail = nlen - p;
        for (int k = 1; k < avail && k <= (int)T.added_max_len; ++k)
          if (cls[p + k] & kHfAddedStart) { avail = k; break; }
        int32_t id;
        al = hf_added_len(T, nb + p, avail, &id, T.n_added_plain, T.n_added);
      }
    }
    uint32_t m = __ballot_sync(kFull, al > 0);
    while (m) {
      const int bit = __ffs(m) - 1;
      m &= m - 1;
      const int q = base + bit;
      const int l = __shfl_sync(kFull, al, bit);
      if (q >= cover) {
        for (int k = lane; k < l; k += 32) cls[q + k] = k == 0 ? kHfAddedStart : kHfInAdded;
        cover = q + l;
        if (!final && q + l > nlen - (int)T.added_max_len && q - 9 < bound) bound = q - 9;
      }
    }
    __syncwarp();
  }
  return bound;
}

// ---- B1 (patterns 1, 2): an apostrophe starts a contraction token iff it is at a token start — i.e. the previous
// char is neither "other" class (the [^\s\p{L}\p{N}]+ run would have swallowed it) nor U+0020 (which is then the " ?"
// prefix of a punctuation run) — and the bytes after it spell one of s t m d re ve ll.  fold: pattern 2's (?i: ...).
__device__ __forceinline__ void hf_mark_contractions(const uint8_t* nb, uint8_t* cls, int nlen, bool fold, int lane) {
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    uint8_t add = 0;
    if (p < nlen && nb[p] == '\'' && !hf_added(cls[p])) {
      bool st = p == 0;
      if (!st) {
        const uint8_t a = cls[hf_char_start(cls, p - 1)];
        st = hf_added(a) || ((a & 3) != kHfOther && !(a & kHfIsSp));
      }
      if (st) {
        uint8_t c1 = (p + 1 < nlen && !hf_added(cls[p + 1])) ? nb[p + 1] : 0;
        uint8_t c2 = (c1 && p + 2 < nlen && !hf_added(cls[p + 2])) ? nb[p + 2] : 0;
        if (fold) {  // ASCII upper case, and U+017F (C5 BF) folds to s
          if (c1 == 0xC5 && c2 == 0xBF) add = kHfContr3;
          if (c1 >= 'A' && c1 <= 'Z') c1 |= 0x20;
          if (c2 >= 'A' && c2 <= 'Z') c2 |= 0x20;
        }
        if (c1 == 's' || c1 == 't' || c1 == 'm' || c1 == 'd') add = kHfContr2;
        else if ((c1 == 'r' && c2 == 'e') || (c1 == 'v' && c2 == 'e') || (c1 == 'l' && c2 == 'l')) add = kHfContr3;
      }
    }
    __syncwarp();
    if (add) cls[p] |= add;
    __syncwarp();
  }
}

// ---- C1, C2 (patterns 2, 3): the facts of a run that the token starts need.  ps (pattern 3): the punctuation whose
// run swallows following CR/LFs is \p{P}|\p{S} rather than the class "other".  Lowers *limit in a non-final buffer to
// the start of a whitespace run that touches its end.
__device__ __forceinline__ void hf_run_facts(const uint8_t* cls, uint8_t* aux, int nlen, int K, bool final, bool ps,
                                             int lane, int* limit) {
  const uint32_t below = (1u << lane) - 1u;
  // ---- C1 (forward): swallowed CR/LFs, digit index inside the run
  bool carry_sw = false;  // the last char that is not CR/LF is a punctuation char
  int carry_d = 0;        // digits since the last non-digit char
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    const uint8_t v = p < nlen ? cls[p] : kHfCont;
    const bool ch = p < nlen && v != kHfCont;                       // a char starts here (added-token bytes count as chars)
    const bool plain = ch && !hf_added(v);
    const bool is_nl = plain && (aux[p] & kAuxNl);
    const bool is_n = plain && (v & 3) == kHfNumber;
    const uint32_t m_o = __ballot_sync(kFull, plain && (ps ? (aux[p < nlen ? p : 0] & kAuxPS) != 0 : (v & 3) == kHfOther));
    const uint32_t m_n = __ballot_sync(kFull, is_n);
    const uint32_t m_not_nl = __ballot_sync(kFull, ch && !is_nl);
    const uint32_t m_not_n = __ballot_sync(kFull, ch && !is_n);
    uint8_t add = 0;
    if (is_nl && hf_last_bit(m_not_nl & below, m_o, carry_sw)) add |= kAuxSwallowed;
    if (is_n && hf_count_after(m_not_n & below, m_n & below, carry_d) % K == 0) add |= kAuxDigitStart;
    if (add) aux[p] |= add;
    carry_sw = hf_last_bit(m_not_nl, m_o, carry_sw);
    carry_d = hf_count_after(m_not_n, m_n, carry_d);
  }
  // ---- C2 (backward): does a CR/LF follow inside the same whitespace run?
  bool carry_nl = false;
  for (int base = ((nlen - 1) >> 5) << 5; base >= 0; base -= 32) {
    const int p = base + lane;
    const uint8_t v = p < nlen ? cls[p] : kHfCont;
    const bool ch = p < nlen && v != kHfCont;
    const bool plain = ch && !hf_added(v);
    const bool is_ws = plain && (v & 3) == kHfSpace;
    const bool is_nl = plain && (aux[p] & kAuxNl);
    const uint32_t m_nl = __ballot_sync(kFull, is_nl);
    const uint32_t m_not_ws = __ballot_sync(kFull, ch && !is_ws);
    if (is_ws && !is_nl) {
      const uint32_t above = ~((2u << lane) - 1u);
      const uint32_t m = m_not_ws & above;
      const uint32_t upto = m ? (above & ((1u << (__ffs(m) - 1)) - 1u)) : above;
      if ((m_nl & upto) || (!m && carry_nl)) aux[p] |= kAuxNlAfter;
    }
    if (m_not_ws) carry_nl = (m_nl & ((1u << (__ffs(m_not_ws) - 1)) - 1u)) != 0;
    else carry_nl = carry_nl || m_nl != 0;
  }
  __syncwarp();
  // a whitespace run that touches the end of a non-final buffer cannot be cut yet (a newline may still come)
  if (!final) {
    const int q = hf_char_start(cls, nlen - 1);
    if (!hf_added(cls[q]) && (cls[q] & 3) == kHfSpace) {
      int run = q;
      for (;;) {
        const int t = hf_char_start(cls, run - 1);
        if (run == 0 || hf_added(cls[t]) || (cls[t] & 3) != kHfSpace || cls[t] == kHfCont) break;
        run = t;
      }
      if (run < *limit) *limit = run;
    }
  }
}

// ---- D1, D2 (pattern 3): "punct + ASCII letters" tokens
__device__ __forceinline__ void hf_ascii_runs(const uint8_t* nb, const uint8_t* cls, uint8_t* aux, int nlen, int lane) {
  // ---- D1: ASCII punctuation that opens a "punct + ASCII letters" token: followed by an ASCII letter, and a token
  // start itself (previous char neither P/S — its run would have taken this one — nor U+0020, the " ?" prefix)
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    bool as = false;
    if (p + 1 < nlen && !hf_added(cls[p]) && hf_ascii_punct(nb[p]) && !hf_added(cls[p + 1]) && hf_ascii_alpha(nb[p + 1])) {
      as = p == 0;
      if (!as) {
        const int q = hf_char_start(cls, p - 1);
        as = hf_added(cls[q]) || (!(aux[q] & kAuxPS) && nb[q] != ' ');
      }
    }
    if (as) aux[p] |= kAuxAStart;
  }
  __syncwarp();
  // ---- D2 (forward): an ASCII letter belongs to such a token iff the nearest preceding char that is not an ASCII
  // letter is one of those openers
  const uint32_t below = (1u << lane) - 1u;
  bool carry_a = false;
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    const uint8_t v = p < nlen ? cls[p] : kHfCont;
    const bool ch = p < nlen && v != kHfCont;
    const bool plain = ch && !hf_added(v);
    const bool alpha = plain && hf_ascii_alpha(nb[p]);
    const uint32_t m_not_alpha = __ballot_sync(kFull, ch && !alpha);
    const uint32_t m_astart = __ballot_sync(kFull, plain && (aux[p < nlen ? p : 0] & kAuxAStart));
    if (alpha && hf_last_bit(m_not_alpha & below, m_astart, carry_a)) aux[p] |= kAuxAIn;
    carry_a = hf_last_bit(m_not_alpha, m_astart, carry_a);
  }
  __syncwarp();
}

// ---- B2: the rules of each pattern for a char at p whose previous char starts at q, outside added tokens and
// contractions.  a non-space char of the same piece follows the char at p (cut: pattern 3, where a number or CJK
// char ends the piece like the end of the text)
__device__ __forceinline__ bool hf_open_next(const uint8_t* nb, const uint8_t* cls, const uint8_t* aux, int nlen, int p,
                                             bool cut) {
  const int nx = p + hf_char_len(nb[p]);
  if (nx >= nlen || (cls[nx] & kHfAddedStart)) return false;
  const uint8_t c = cls[nx] & 3;
  return c != kHfSpace && !(cut && (c == kHfNumber || (aux[nx] & kAuxCjk)));
}

// pattern 1: whitespace after non-whitespace | whitespace that is the LAST of a run of >= 2 followed by a non-space in
// the same segment (the \s+(?!\S) backtrack) | non-whitespace after whitespace other than U+0020 (a single U+0020 is
// the " ?" prefix) | class change between two non-whitespace chars
__device__ __forceinline__ bool hf_rules1(const uint8_t* nb, const uint8_t* cls, int nlen, int p, int q) {
  const uint8_t v = cls[p], a = cls[q];
  const bool a_ws = (a & 3) == kHfSpace;
  if ((v & 3) == kHfSpace) return !a_ws || hf_open_next(nb, cls, nullptr, nlen, p, false);
  return a_ws ? !(a & kHfIsSp) : (a & 3) != (v & 3);
}

// whitespace of patterns 2 and 3: CR/LF: not swallowed and the previous char is not whitespace; other whitespace: run
// start | previous char is a swallowed CR/LF while a newline still follows in the run, else previous char is a CR/LF
// or this is the last char of the run before a non-space (prefix or single)
__device__ __forceinline__ bool hf_rules_ws(const uint8_t* nb, const uint8_t* cls, const uint8_t* aux, int nlen, int p,
                                            int q, bool cut) {
  const bool a_ws = (cls[q] & 3) == kHfSpace;
  const uint8_t a_aux = aux[q], b_aux = aux[p];
  if (b_aux & kAuxNl) return !(b_aux & kAuxSwallowed) && !a_ws;
  if (b_aux & kAuxNlAfter) return !a_ws || ((a_aux & kAuxNl) && (a_aux & kAuxSwallowed));
  return !a_ws || (a_aux & kAuxNl) || hf_open_next(nb, cls, aux, nlen, p, cut);
}

// pattern 2:
//   letter: the previous char is a number or CR/LF, or a punctuation char that is NOT itself a token start (a
//           punctuation / space / tab char that IS a token start is the letters' one-char prefix);
//   number: index in the digit run is a multiple of K;      punctuation: previous char is neither punctuation nor U+0020;
//   whitespace: hf_rules_ws
__device__ __forceinline__ bool hf_rules2(const uint8_t* nb, const uint8_t* cls, const uint8_t* aux, int nlen, int p, int q) {
  const uint8_t v = cls[p], a = cls[q];
  const uint8_t bc = v & 3, ac = a & 3;
  if (bc == kHfLetter) {
    if (ac == kHfLetter) return false;
    if (ac == kHfNumber) return true;
    if (ac == kHfSpace) return (aux[q] & kAuxNl) != 0;   // a space / tab is the letters' prefix, a newline is not
    // punctuation before letters: it is their prefix iff it is a token start itself
    bool a_start = q == 0 || hf_added(cls[q - 1]);
    if (!a_start) {
      const uint8_t t = cls[hf_char_start(cls, q - 1)];
      a_start = (t & 3) != kHfOther && !(t & kHfIsSp);
    }
    return !a_start;
  }
  if (bc == kHfNumber) return (aux[p] & kAuxDigitStart) != 0;
  if (bc == kHfOther) return ac != kHfOther && !(a & kHfIsSp);
  return hf_rules_ws(nb, cls, aux, nlen, p, q, false);
}

// pattern 3.  Kinds: letter (\p{L} or \p{M}), number, CJK, whitespace, P/S, rest.
//   number: index in the run is a multiple of 3;   CJK: previous char is not CJK;   anything after a number / CJK char;
//   letter: after a letter only where a "punct + ASCII letters" token ends (this char is not an ASCII letter); after
//           P/S unless that char opens such a token and this is an ASCII letter; after whitespace only if it is a CR/LF
//           (any other whitespace or "rest" char is the letters' one-char prefix);
//   P/S   : previous char is neither P/S nor U+0020;
//   rest  : previous char is not "rest", or a letter follows (then this char is the letters' prefix);
//   whitespace: hf_rules_ws, where a following number / CJK char ends the piece like the end of the text.
__device__ __forceinline__ bool hf_rules3(const uint8_t* nb, const uint8_t* cls, const uint8_t* aux, int nlen, int p, int q) {
  const uint8_t v = cls[p], a = cls[q], b_aux = aux[p], a_aux = aux[q];
  const uint8_t bc = v & 3, ac = a & 3;
  if (bc == kHfNumber) return (b_aux & kAuxDigitStart) != 0;
  if (b_aux & kAuxCjk) return !(a_aux & kAuxCjk);
  if (ac == kHfNumber || (a_aux & kAuxCjk)) return true;         // the previous char closed a piece
  if (bc == kHfLetter) {
    if (ac == kHfLetter) return (a_aux & kAuxAIn) && !hf_ascii_alpha(nb[p]);
    if (a_aux & kAuxPS) return !((a_aux & kAuxAStart) && hf_ascii_alpha(nb[p]));
    if (ac == kHfSpace) return (a_aux & kAuxNl) != 0;
    return false;                                                 // a "rest" char is the letters' prefix
  }
  if (b_aux & kAuxPS) return !(a_aux & kAuxPS) && !(a & kHfIsSp);
  if (bc == kHfOther) {                                           // "rest": control / format / unassigned
    const int nx = p + hf_char_len(nb[p]);
    const bool a_rest = ac == kHfOther && !(a_aux & (kAuxPS | kAuxCjk));
    return !a_rest || (nx < nlen && !hf_added(cls[nx]) && (cls[nx] & 3) == kHfLetter);
  }
  return hf_rules_ws(nb, cls, aux, nlen, p, q, true);
}

// ---- B2: does a token start at p?  Buffer / segment start, added token, contraction start; never inside an added
// token or a contraction, always right after one; otherwise the model's rules.
__device__ __forceinline__ bool hf_token_start(int pattern, const uint8_t* nb, const uint8_t* cls, const uint8_t* aux,
                                               int nlen, int p) {
  const uint8_t v = cls[p];
  if (v == kHfCont || v == kHfInAdded) return false;
  if (p == 0 || (v & kHfAddedStart) || hf_added(cls[p - 1]) || (v & kHfContr)) return true;
  const uint8_t c1 = cls[p - 1] & kHfContr, c2 = p >= 2 ? (cls[p - 2] & kHfContr) : 0, c3 = p >= 3 ? (cls[p - 3] & kHfContr) : 0;
  if (c1 || c2 == kHfContr3) return false;              // inside a contraction
  if (c2 == kHfContr2 || c3 == kHfContr3) return true;   // right after one
  const int q = hf_char_start(cls, p - 1);
  if (pattern == 3) return hf_rules3(nb, cls, aux, nlen, p, q);
  if (pattern == 2) return hf_rules2(nb, cls, aux, nlen, p, q);
  return hf_rules1(nb, cls, nlen, p, q);
}

// nb[0..nlen) starts at a token start.  final: the text ends at nlen.  TWO: the model's added tokens are matched in
// two passes (normalized:false, then normalized:true between those).
template <bool TWO, typename SM>
__device__ HfScan hf_scan(const SpDev& T, SM& sm, int nlen, bool final, int lane) {
  const uint8_t* nb = sm.nbuf;
  uint8_t* cls = reinterpret_cast<uint8_t*>(sm.S);
  uint8_t* aux = reinterpret_cast<uint8_t*>(sm.PM);
  static_assert(sizeof(sm.S) >= kNBuf && sizeof(sm.PM) >= kNBuf, "class scratch must cover the staging buffer");
  HfScan r;
  r.nwords = 0;
  r.tail_start = 0;
  r.capped = false;
  // T.hf_pattern is read from the kernel parameters at each use: a local copy kept live across the passes costs the
  // HF kernels registers
  r.bad = hf_classify(T, nb, cls, aux, nlen, final, T.hf_pattern, lane);
  if (r.bad) return r;
  int bound = nlen;
  if constexpr (TWO) {
    hf_mark_added(T, nb, cls, nlen, T.n_added_plain, lane);
    bound = hf_mark_added_second(T, nb, cls, nlen, final, lane);
  } else if (T.n_added) {
    hf_mark_added(T, nb, cls, nlen, T.n_added, lane);
  }
  if (T.hf_pattern != 3) hf_mark_contractions(nb, cls, nlen, T.hf_pattern == 2, lane);
  // non-final: a token is complete only if everything that decides its end is in the buffer
  int limit = final ? nlen : nlen - (int)T.added_max_len - 8;
  if constexpr (TWO) limit = min(limit, bound);
  if (T.hf_pattern == 2 || T.hf_pattern == 3) hf_run_facts(cls, aux, nlen, T.hf_digits, final, T.hf_pattern == 3, lane, &limit);
  if (T.hf_pattern == 3) hf_ascii_runs(nb, cls, aux, nlen, lane);
  // ---- B2: token starts, compacted into wstart[]
  constexpr int kCap = kMaxWords - 1;
  int count = 0;
  for (int base = 0; base < nlen && base <= limit && !r.capped; base += 32) {
    const int p = base + lane;
    const bool in = p < nlen && p <= limit;
    const bool special = in && (cls[p] & kHfAddedStart);
    const bool st = in && hf_token_start(T.hf_pattern, nb, cls, aux, nlen, p);
    const uint32_t m = __ballot_sync(kFull, st);
    const int idx = count + __popc(m & ((1u << lane) - 1));
    if (st && idx < kCap) sm.wstart[idx] = (uint16_t)(p | (special ? kHfSpecialWord : 0));
    count += __popc(m);
    if (count >= kCap) { count = kCap; r.capped = true; }
  }
  __syncwarp();
  if (final && !r.capped) {
    r.nwords = count;
    r.tail_start = nlen;
    if (lane == 0) sm.wstart[count] = (uint16_t)nlen;
  } else if (count == 0) {
    r.nwords = 0;
    r.tail_start = 0;
  } else {
    // the last start listed opens the first token that is not known to be complete
    r.nwords = count - 1;
    r.tail_start = sm.wstart[count - 1] & kHfPosMask;
  }
  __syncwarp();
  return r;
}
