// hf_pretok.cuh — warp-parallel pre-tokenizer of the HF byte-level BPE backend (included by sp_encode.cu).
//
// Device replacement for the two steps the Rust crate runs before BPE inside tokenizers_encode
// (xllm_service/tokenizer/tokenizers/src/lib.rs:83-99 -> Tokenizer::encode):
//   added_vocabulary.rs   split the text on the added (special) tokens, leftmost-longest, verbatim
//   pre_tokenizers/byte_level.rs   split every remaining segment with the GPT-2 pattern
//        's|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+
// (the oracle's sequential restatement: oracle/hf_bpe_oracle.cc gpt2_split).
//
// The leftmost-first regex scan is sequential as written, but every token boundary of THIS pattern is decided by
// a window of one char back, one char ahead (plus two ASCII bytes after an apostrophe), so the warp decides all
// positions of the staging buffer at once:
//   A   class of every char (letter / number / whitespace / other, Unicode tables), UTF-8 validation
//   A2  added-token starts (first-byte filter, then compare), resolved leftmost-longest / non-overlapping
//   B1  an apostrophe starts a contraction token iff it is at a token start — i.e. the previous char is neither
//       "other" class (the [^\s\p{L}\p{N}]+ run would have swallowed it) nor U+0020 (which is then the " ?" prefix
//       of a punctuation run) — and the bytes after it spell one of s t m d re ve ll
//   B2  position i starts a token iff: segment start | contraction start | contraction end | (not inside a
//       contraction and)  whitespace after non-whitespace | whitespace that is the LAST of a run of >= 2 followed
//       by a non-space in the same segment (the \s+(?!\S) backtrack) | non-whitespace after whitespace other
//       than U+0020 (a single U+0020 is the " ?" prefix) | class change between two non-whitespace chars.
// hf_pattern 2 is the cl100k-family Split regex of the newer layouts (Llama-3: K = 3, Qwen2: K = 1)
//        (?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,K}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
// (oracle: cl100k_split).  Still decided per position, with three facts that need a scan along the buffer, done
// 32 bytes at a time with a warp-uniform carry: C1 forward — a CR/LF is "swallowed" when only CR/LFs separate it
// from a punctuation char (the [\r\n]* tail of the punctuation alternative), and a digit's index inside its run
// (a token starts every K digits); C2 backward — a non-newline whitespace char has a CR/LF later in its
// whitespace run (then \s*[\r\n]+ takes the run up to the LAST newline).  With those, position i starts a token iff
//   letter: the previous char is a number or CR/LF, or a punctuation char that is NOT itself a token start (a
//           punctuation / space / tab char that IS a token start is the letters' one-char prefix);
//   number: index in the digit run is a multiple of K;      punctuation: previous char is neither punctuation nor U+0020;
//   CR/LF : not swallowed and the previous char is not whitespace;
//   other whitespace: run start | previous char is a CR/LF with no newline left in the run | last char of the run
//           before a non-space (prefix or single) — and nothing else while a newline still follows in the run;
// contractions are case-insensitive (incl. U+017F) and otherwise as above.
// hf_pattern 3 is DeepSeek-V3 / R1: Sequence[Split(\p{N}{1,3}), Split([一-龥぀-ゟ゠-ヿ]+), Split(main regex)], all Isolated —
// numbers (groups of 3) and CJK / kana runs are cut out first and bound everything else; inside the remaining pieces
//        [!-/:-@\[-`{-~][A-Za-z]+|[^\r\n\p{L}\p{P}\p{S}]?[\p{L}\p{M}]+| ?[\p{P}\p{S}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
// (oracle: ds3_split; the rule set below is checked against the sequential scan in tests/test_hf_rules_equivalence.py).
// Kinds: letter (\p{L} or \p{M}), number, CJK, whitespace, P/S, rest.  The scanned facts of pattern 2 carry over (with
// "punctuation" = P/S) plus one more forward scan: an ASCII letter lies inside a "punct + ASCII letters" token when
// the nearest preceding char that is not an ASCII letter is an ASCII punctuation char that starts a token and is
// followed by an ASCII letter.  Position i starts a token iff
//   number: index in the run is a multiple of 3;   CJK: previous char is not CJK;   anything after a number / CJK char;
//   letter: after a letter only where a "punct + ASCII letters" token ends (this char is not an ASCII letter); after
//           P/S unless that char opens such a token and this is an ASCII letter; after whitespace only if it is a CR/LF
//           (any other whitespace or "rest" char is the letters' one-char prefix);
//   P/S   : previous char is neither P/S nor U+0020;
//   rest  : previous char is not "rest", or a letter follows (then this char is the letters' prefix);
//   whitespace: as in pattern 2, where a following number / CJK char ends the piece like the end of the text.
// Per-byte scratch (one byte per text byte, in the merge scratch S[] which is idle while scanning):
//   bits 0-1 class, bit 2 char is U+0020, bit 3 inside an added token, bit 4 added token starts here,
//   bits 5-6 contraction length - 1 (0 = none), 0x80 = UTF-8 continuation byte.
#pragma once

enum : uint8_t { kHfOther = 0, kHfLetter = 1, kHfNumber = 2, kHfSpace = 3 };
constexpr uint8_t kHfIsSp = 0x04, kHfInAdded = 0x08, kHfAddedStart = 0x10, kHfCont = 0x80;
constexpr uint16_t kHfSpecialWord = 0x8000;  // wstart[] flag: the word is an added token (one id, no BPE)
constexpr uint16_t kHfPosMask = 0x0FFF;
// pattern 2, second scratch byte per text byte (in PM[]): CR/LF | swallowed CR/LF | digit starts a token | a CR/LF follows in the run
constexpr uint8_t kAuxNl = 0x01, kAuxSwallowed = 0x02, kAuxDigitStart = 0x04, kAuxNlAfter = 0x08;
// pattern 3 (DeepSeek-V3), same byte: \p{P}|\p{S} char | char of the CJK / kana ranges | ASCII punctuation that opens a
// "punct + ASCII letters" token | ASCII letter inside such a token
constexpr uint8_t kAuxPS = 0x10, kAuxCjk = 0x20, kAuxAStart = 0x40, kAuxAIn = 0x80;
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

// longest added token that is a prefix of p[0..avail); 0 = none.  *id = its token id.
__device__ __forceinline__ int hf_added_len(const SpDev& T, const uint8_t* p, int avail, int32_t* id) {
  int best = 0;
  for (uint32_t a = 0; a < T.n_added; ++a) {
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

// nb[0..nlen) starts at a token start.  cls = nlen bytes of scratch.  final: the text ends at nlen.
template <typename SM>
__device__ HfScan hf_scan(const SpDev& T, SM& sm, int nlen, bool final, int lane) {
  const uint8_t* nb = sm.nbuf;
  uint8_t* cls = reinterpret_cast<uint8_t*>(sm.S);
  uint8_t* aux = reinterpret_cast<uint8_t*>(sm.PM);
  static_assert(sizeof(sm.S) >= kNBuf && sizeof(sm.PM) >= kNBuf, "class scratch must cover the staging buffer");
  const bool p2 = T.hf_pattern == 2, p3 = T.hf_pattern == 3;
  bool bad = false, nfc_bad = false;
  // ---- A: classes + UTF-8 validation (+ the NFC quick check: every char NFC-inert => NFC is the identity)
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
          cov = (x >= 0xF0 ? 4 : (x >= 0xE0 ? 3 : (x >= 0xC0 ? 2 : 1))) > k;
          break;
        }
        bad |= !cov;
      } else {
        const int l = b0 >= 0xF0 ? 4 : (b0 >= 0xE0 ? 3 : 2);
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
      if (p2 || p3) aux[p] = ax;
    }
  }
  __syncwarp();
  HfScan r;
  r.nwords = 0;
  r.tail_start = 0;
  r.capped = false;
  r.bad = __any_sync(kFull, bad) ? 1 : (__any_sync(kFull, nfc_bad) ? 2 : 0);
  if (r.bad) return r;
  // ---- A2: added tokens, leftmost-longest, non-overlapping
  if (T.n_added) {
    int cover = 0;
    for (int base = 0; base < nlen; base += 32) {
      const int p = base + lane;
      int al = 0;
      if (p < nlen) {
        const uint8_t b0 = nb[p];
        if ((T.added_first[b0 >> 5] >> (b0 & 31)) & 1u) {
          int32_t id;
          al = hf_added_len(T, nb + p, nlen - p, &id);
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
  // ---- B1: contraction starts
  for (int base = 0; base < nlen; base += 32) {
    const int p = base + lane;
    uint8_t add = 0;
    if (!p3 && p < nlen && nb[p] == '\'' && !(cls[p] & (kHfInAdded | kHfAddedStart))) {
      bool st = p == 0;
      if (!st) {
        int q = p - 1;
        while (q > 0 && cls[q] == kHfCont) --q;
        const uint8_t a = cls[q];
        st = (a & (kHfInAdded | kHfAddedStart)) || ((a & 3) != kHfOther && !(a & kHfIsSp));
      }
      if (st) {
        uint8_t c1 = (p + 1 < nlen && !(cls[p + 1] & (kHfInAdded | kHfAddedStart))) ? nb[p + 1] : 0;
        uint8_t c2 = (c1 && p + 2 < nlen && !(cls[p + 2] & (kHfInAdded | kHfAddedStart))) ? nb[p + 2] : 0;
        if (p2) {  // (?i: ...): ASCII upper case, and U+017F (C5 BF) folds to s
          if (c1 == 0xC5 && c2 == 0xBF) add = 0x40;
          if (c1 >= 'A' && c1 <= 'Z') c1 |= 0x20;
          if (c2 >= 'A' && c2 <= 'Z') c2 |= 0x20;
        }
        if (c1 == 's' || c1 == 't' || c1 == 'm' || c1 == 'd') add = 0x20;
        else if ((c1 == 'r' && c2 == 'e') || (c1 == 'v' && c2 == 'e') || (c1 == 'l' && c2 == 'l')) add = 0x40;
      }
    }
    __syncwarp();
    if (add) cls[p] |= add;
    __syncwarp();
  }
  // non-final: a token is complete only if everything that decides its end is in the buffer
  int limit = final ? nlen : nlen - (int)T.added_max_len - 8;
  if (p2 || p3) {
    const uint32_t below = (1u << lane) - 1u;
    // ---- C1 (forward): swallowed CR/LFs, digit index inside the run
    bool carry_sw = false;  // the last char that is not CR/LF is a punctuation char
    int carry_d = 0;        // digits since the last non-digit char
    const int K = T.hf_digits;
    for (int base = 0; base < nlen; base += 32) {
      const int p = base + lane;
      const uint8_t v = p < nlen ? cls[p] : kHfCont;
      const bool ch = p < nlen && v != kHfCont;                       // a char starts here (added-token bytes count as chars)
      const bool plain = ch && !(v & (kHfInAdded | kHfAddedStart));
      const bool is_nl = plain && (aux[p] & kAuxNl);
      const bool is_n = plain && (v & 3) == kHfNumber;
      // the char class whose run swallows following CR/LFs: pattern 2 [^\s\p{L}\p{N}], pattern 3 [\p{P}\p{S}]
      const uint32_t m_o = __ballot_sync(kFull, plain && (p3 ? (aux[p < nlen ? p : 0] & kAuxPS) != 0 : (v & 3) == kHfOther));
      const uint32_t m_n = __ballot_sync(kFull, is_n);
      const uint32_t m_not_nl = __ballot_sync(kFull, ch && !is_nl);
      const uint32_t m_not_n = __ballot_sync(kFull, ch && !is_n);
      uint8_t add = 0;
      if (is_nl) {
        const uint32_t m = m_not_nl & below;
        if (m ? ((m_o >> (31 - __clz(m))) & 1u) : (uint32_t)carry_sw) add |= kAuxSwallowed;
      }
      if (is_n) {
        const uint32_t m = m_not_n & below;
        const int idx = m ? __popc(m_n & below & ~((2u << (31 - __clz(m))) - 1u)) : carry_d + __popc(m_n & below);
        if (idx % K == 0) add |= kAuxDigitStart;
      }
      if (add) aux[p] |= add;
      if (m_not_nl) carry_sw = (m_o >> (31 - __clz(m_not_nl))) & 1u;
      if (m_not_n) carry_d = __popc(m_n & ~((2u << (31 - __clz(m_not_n))) - 1u));
      else carry_d += __popc(m_n);
    }
    // ---- C2 (backward): does a CR/LF follow inside the same whitespace run?
    bool carry_nl = false;
    for (int base = ((nlen - 1) >> 5) << 5; base >= 0; base -= 32) {
      const int p = base + lane;
      const uint8_t v = p < nlen ? cls[p] : kHfCont;
      const bool ch = p < nlen && v != kHfCont;
      const bool plain = ch && !(v & (kHfInAdded | kHfAddedStart));
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
      int q = nlen - 1;
      while (q > 0 && cls[q] == kHfCont) --q;
      if (!(cls[q] & (kHfInAdded | kHfAddedStart)) && (cls[q] & 3) == kHfSpace) {
        int run = q;
        for (;;) {
          int t = run - 1;
          while (t > 0 && cls[t] == kHfCont) --t;
          if (run == 0 || (cls[t] & (kHfInAdded | kHfAddedStart)) || (cls[t] & 3) != kHfSpace || cls[t] == kHfCont) break;
          run = t;
        }
        if (run < limit) limit = run;
      }
    }
  }
  if (p3) {
    // ---- D1: ASCII punctuation that opens a "punct + ASCII letters" token: followed by an ASCII letter, and a token
    // start itself (previous char neither P/S — its run would have taken this one — nor U+0020, the " ?" prefix)
    for (int base = 0; base < nlen; base += 32) {
      const int p = base + lane;
      bool as = false;
      if (p + 1 < nlen && !(cls[p] & (kHfInAdded | kHfAddedStart)) && hf_ascii_punct(nb[p]) &&
          !(cls[p + 1] & (kHfInAdded | kHfAddedStart)) && hf_ascii_alpha(nb[p + 1])) {
        as = p == 0;
        if (!as) {
          int q = p - 1;
          while (q > 0 && cls[q] == kHfCont) --q;
          as = (cls[q] & (kHfInAdded | kHfAddedStart)) || (!(aux[q] & kAuxPS) && nb[q] != ' ');
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
      const bool plain = ch && !(v & (kHfInAdded | kHfAddedStart));
      const bool alpha = plain && hf_ascii_alpha(nb[p]);
      const uint32_t m_not_alpha = __ballot_sync(kFull, ch && !alpha);
      const uint32_t m_astart = __ballot_sync(kFull, plain && (aux[p < nlen ? p : 0] & kAuxAStart));
      if (alpha) {
        const uint32_t m = m_not_alpha & below;
        if (m ? ((m_astart >> (31 - __clz(m))) & 1u) : (uint32_t)carry_a) aux[p] |= kAuxAIn;
      }
      if (m_not_alpha) carry_a = (m_astart >> (31 - __clz(m_not_alpha))) & 1u;
    }
    __syncwarp();
  }
  // ---- B2: token starts, compacted into wstart[]
  constexpr int kCap = kMaxWords - 1;
  int count = 0;
  for (int base = 0; base < nlen && base <= limit && !r.capped; base += 32) {
    const int p = base + lane;
    bool st = false, special = false;
    if (p < nlen && p <= limit) {
      const uint8_t v = cls[p];
      if (v == kHfCont || v == kHfInAdded) {
        st = false;
      } else if (v & kHfAddedStart) {
        st = special = true;
      } else if (p == 0 || (cls[p - 1] & (kHfInAdded | kHfAddedStart)) || (v & 0x60)) {
        st = true;  // buffer / segment start, contraction start
      } else {
        const uint8_t c1 = cls[p - 1] & 0x60, c2 = p >= 2 ? (cls[p - 2] & 0x60) : 0, c3 = p >= 3 ? (cls[p - 3] & 0x60) : 0;
        if (c1 || c2 == 0x40) st = false;              // inside a contraction
        else if (c2 == 0x20 || c3 == 0x40) st = true;   // right after one
        else {
          int q = p - 1;
          while (q > 0 && cls[q] == kHfCont) --q;
          const uint8_t a = cls[q];
          const bool a_ws = (a & 3) == kHfSpace, b_ws = (v & 3) == kHfSpace;
          if (p3) {
            const uint8_t a_aux = aux[q], b_aux = aux[p];
            const uint8_t bc = v & 3, ac = a & 3;
            const bool a_bound = ac == kHfNumber || (a_aux & kAuxCjk);     // the previous char closed a piece
            if (bc == kHfNumber) {
              st = (b_aux & kAuxDigitStart) != 0;
            } else if (b_aux & kAuxCjk) {
              st = !(a_aux & kAuxCjk);
            } else if (a_bound) {
              st = true;
            } else if (bc == kHfLetter) {
              if (ac == kHfLetter) st = (a_aux & kAuxAIn) && !hf_ascii_alpha(nb[p]);
              else if (a_aux & kAuxPS) st = !((a_aux & kAuxAStart) && hf_ascii_alpha(nb[p]));
              else if (a_ws) st = (a_aux & kAuxNl) != 0;
              else st = false;                                             // a "rest" char is the letters' prefix
            } else if (b_aux & kAuxPS) {
              st = !(a_aux & kAuxPS) && !(a & kHfIsSp);
            } else if (bc == kHfOther) {                                   // "rest": control / format / unassigned
              const uint8_t b0 = nb[p];
              const int nx = p + (b0 < 0x80 ? 1 : (b0 < 0xE0 ? 2 : (b0 < 0xF0 ? 3 : 4)));
              const bool a_rest = ac == kHfOther && !(a_aux & (kAuxPS | kAuxCjk));
              st = !a_rest || (nx < nlen && !(cls[nx] & (kHfInAdded | kHfAddedStart)) && (cls[nx] & 3) == kHfLetter);
            } else if (b_aux & kAuxNl) {
              st = !(b_aux & kAuxSwallowed) && !a_ws;
            } else if (b_aux & kAuxNlAfter) {
              st = !a_ws || ((a_aux & kAuxNl) && (a_aux & kAuxSwallowed));
            } else {
              const uint8_t b0 = nb[p];
              const int nx = p + (b0 < 0x80 ? 1 : (b0 < 0xE0 ? 2 : (b0 < 0xF0 ? 3 : 4)));
              // a non-space char of the same piece follows (a number / CJK char ends the piece like the end of text)
              const bool nxt_open = nx < nlen && !(cls[nx] & kHfAddedStart) && (cls[nx] & 3) != kHfSpace &&
                                    (cls[nx] & 3) != kHfNumber && !(aux[nx] & kAuxCjk);
              st = !a_ws || (a_aux & kAuxNl) || nxt_open;
            }
          } else if (p2) {
            const uint8_t a_aux = aux[q], b_aux = aux[p];
            const uint8_t bc = v & 3, ac = a & 3;
            if (bc == kHfLetter) {
              if (ac == kHfLetter) st = false;
              else if (ac == kHfNumber) st = true;
              else if (a_ws) st = (a_aux & kAuxNl) != 0;   // a space / tab is the letters' prefix, a newline is not
              else {
                // punctuation before letters: it is their prefix iff it is a token start itself
                bool a_start = q == 0 || (cls[q - 1] & (kHfInAdded | kHfAddedStart));
                if (!a_start) {
                  int t = q - 1;
                  while (t > 0 && cls[t] == kHfCont) --t;
                  a_start = (cls[t] & 3) != kHfOther && !(cls[t] & kHfIsSp);
                }
                st = !a_start;
              }
            } else if (bc == kHfNumber) {
              st = (b_aux & kAuxDigitStart) != 0;
            } else if (bc == kHfOther) {
              st = ac != kHfOther && !(a & kHfIsSp);
            } else if (b_aux & kAuxNl) {
              st = !(b_aux & kAuxSwallowed) && !a_ws;
            } else if (b_aux & kAuxNlAfter) {
              st = !a_ws || ((a_aux & kAuxNl) && (a_aux & kAuxSwallowed));
            } else {
              const uint8_t b0 = nb[p];
              const int nx = p + (b0 < 0x80 ? 1 : (b0 < 0xE0 ? 2 : (b0 < 0xF0 ? 3 : 4)));
              st = !a_ws || (a_aux & kAuxNl) ||
                   (nx < nlen && !(cls[nx] & kHfAddedStart) && (cls[nx] & 3) != kHfSpace);
            }
          } else if (b_ws) {
            if (!a_ws) st = true;
            else {
              const uint8_t b0 = nb[p];
              const int nx = p + (b0 < 0x80 ? 1 : (b0 < 0xE0 ? 2 : (b0 < 0xF0 ? 3 : 4)));
              st = nx < nlen && !(cls[nx] & kHfAddedStart) && (cls[nx] & 3) != kHfSpace;
            }
          } else {
            st = a_ws ? !(a & kHfIsSp) : ((a & 3) != (v & 3));
          }
        }
      }
    }
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
