// oracle/hf_bpe_oracle.cc -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// CPU restatement of the reference's HF-tokenizers backend for byte-level BPE `tokenizer.json` models:
//   xllm_service/tokenizer/tokenizer_factory.cpp:14-19    tokenizer.json present -> FastTokenizer
//   xllm_service/tokenizer/fast_tokenizer.cpp:20-30       encode = tokenizers_encode(text, add_special_tokens = 1); REPLACES *ids
//   xllm_service/tokenizer/tokenizers/src/lib.rs:38-41,83-99   Tokenizer::encode(text, add_special_tokens)
// The arithmetic is the Rust crate `tokenizers` 0.21 (Cargo.toml:11, absent from the reference checkout); this file
// restates its published pipeline for the configuration GPT-2 style models use:
//   added_vocabulary.rs   text is first split on the added tokens that are not `normalized`, leftmost-longest; the
//                         `normalized` ones are then matched the same way inside the pieces between those
//   pre_tokenizers/byte_level.rs   regex split
//        's|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+   then bytes -> GPT-2 byte chars
//   pre_tokenizers/split.rs + byte_level.rs(use_regex = false)   the newer layout (Llama-3, Qwen2, OLMo-2 ...):
//        Split(Regex, Isolated) with the cl100k-family pattern
//        (?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,K}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
//        (K = 3 for Llama-3, plain \p{N} i.e. K = 1 for Qwen2), then the byte alphabet
//   models/bpe/model.rs   ignore_merges: a pre-token that is itself in the vocabulary is emitted as that id
//   models/bpe/word.rs    merge_all: lowest merge rank first, leftmost on ties
// Pinned against pip `tokenizers` 0.22.2 by tests/test_oracle_hf.py (committed goldens
// tests/golden/hf_bpe_goldens.json + live fuzz).  The vocabulary / merges are handed over by the test
// harness (it reads tokenizer.json with Python's json), so no JSON parser lives here.
#include <stdint.h>
#include <string.h>

#include <queue>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

namespace {

#include "unicode_classes.inc"

enum { kOther = 0, kLetter = 1, kNumber = 2, kSpace = 3 };
inline int uni_class(uint32_t cp) {
  if (cp >= 0x110000) return kOther;
  return kUniStage2[(size_t)kUniStage1[cp >> 8] * 256 + (cp & 255)] & 3;  // bit 2: NFC-suspect (unused here)
}
// what a class-0 ("other") char is: 1 = \p{P}, 2 = \p{S}, 3 = \p{M}, 0 = the rest (C*, unassigned ...)
enum { kSubNone = 0, kSubP = 1, kSubS = 2, kSubM = 3 };
int uni_sub(uint32_t cp) {
  if (cp >= 0x110000) return kSubNone;
  return (kUniStage2[(size_t)kUniStage1[cp >> 8] * 256 + (cp & 255)] >> 3) & 3;
}

struct Hf {
  int32_t byte_sym[256];                                   // byte -> id of its byte-level char
  std::unordered_map<uint64_t, std::pair<uint32_t, int32_t>> merges;  // (a << 32 | b) -> (rank, new id)
  std::vector<std::pair<std::string, int32_t>> added;      // added tokens matched on the raw text
  std::vector<bool> added_normalized;                      // normalized: matched in the second pass only
  int pattern = 1;                                         // 1: GPT-2 ByteLevel regex, 2: cl100k family, 3: DeepSeek-V3
  int digits = 3;                                          // pattern 2: \p{N}{1,digits}
  bool ignore_merges = false;
  std::unordered_map<std::string, int32_t> vocab;          // raw bytes of every token -> id (ignore_merges)
};

// strict UTF-8 decode; returns length or 0 when malformed (Rust &str cannot hold malformed text:
// lib.rs:91 unwraps from_utf8 and panics)
int decode(const uint8_t* p, size_t avail, uint32_t* cp) {
  const uint8_t b0 = p[0];
  if (b0 < 0x80) { *cp = b0; return 1; }
  auto tr = [](uint8_t x) { return (x & 0xC0) == 0x80; };
  if ((b0 & 0xE0) == 0xC0 && avail >= 2 && tr(p[1])) {
    *cp = ((b0 & 0x1F) << 6) | (p[1] & 0x3F);
    return *cp >= 0x80 ? 2 : 0;
  }
  if ((b0 & 0xF0) == 0xE0 && avail >= 3 && tr(p[1]) && tr(p[2])) {
    *cp = ((b0 & 0x0F) << 12) | ((p[1] & 0x3F) << 6) | (p[2] & 0x3F);
    return (*cp >= 0x800 && !(*cp >= 0xD800 && *cp < 0xE000)) ? 3 : 0;
  }
  if ((b0 & 0xF8) == 0xF0 && avail >= 4 && tr(p[1]) && tr(p[2]) && tr(p[3])) {
    *cp = ((b0 & 0x07) << 18) | ((p[1] & 0x3F) << 12) | ((p[2] & 0x3F) << 6) | (p[3] & 0x3F);
    return (*cp >= 0x10000 && *cp <= 0x10FFFF) ? 4 : 0;
  }
  return 0;
}

struct Ch {
  uint32_t cp;
  int cls;
  uint32_t off, len;
};

// The ByteLevel regex, alternative by alternative (leftmost-first; each alternative greedy).
// chars: decoded text.  Returns piece boundaries as indices into chars.
void gpt2_split(const std::vector<Ch>& c, std::vector<std::pair<size_t, size_t>>* out) {
  const size_t n = c.size();
  size_t i = 0;
  auto is = [&](size_t k, uint32_t ch) { return k < n && c[k].cp == ch; };
  while (i < n) {
    size_t j = i;
    // 's|'t|'re|'ve|'m|'ll|'d
    if (c[i].cp == '\'') {
      if (is(i + 1, 's') || is(i + 1, 't') || is(i + 1, 'm') || is(i + 1, 'd')) j = i + 2;
      else if ((is(i + 1, 'r') && is(i + 2, 'e')) || (is(i + 1, 'v') && is(i + 2, 'e')) || (is(i + 1, 'l') && is(i + 2, 'l'))) j = i + 3;
    }
    if (j == i) {
      // " ?\p{L}+" | " ?\p{N}+" | " ?[^\s\p{L}\p{N}]+"
      const size_t s = (c[i].cp == ' ' && i + 1 < n && c[i + 1].cls != kSpace) ? i + 1 : i;
      if (c[s].cls != kSpace) {
        const int k = c[s].cls;
        j = s;
        while (j < n && c[j].cls == k) ++j;
      }
    }
    if (j == i) {
      // "\s+(?!\S)" | "\s+"
      size_t e = i;
      while (e < n && c[e].cls == kSpace) ++e;
      if (e == n) j = e;              // run reaches the end: (?!\S) holds after the whole run
      else if (e - i >= 2) j = e - 1; // backtrack one char so that a space follows
      else j = e;                     // single whitespace before a non-space: plain \s+
    }
    out->emplace_back(i, j);
    i = j;
  }
}

inline bool is_nl(uint32_t cp) { return cp == '\r' || cp == '\n'; }
inline uint32_t fold(uint32_t cp) {  // the simple case folds that can hit the contraction letters
  if (cp >= 'A' && cp <= 'Z') return cp + 32;
  if (cp == 0x17F) return 's';  // LATIN SMALL LETTER LONG S folds to s
  return cp;
}

// The cl100k-family pattern, alternative by alternative (leftmost-first, each alternative greedy with backtracking
// exactly where the pattern allows it).
void cl100k_split(const std::vector<Ch>& c, int K, std::vector<std::pair<size_t, size_t>>* out) {
  const size_t n = c.size();
  size_t i = 0;
  auto isf = [&](size_t k, uint32_t ch) { return k < n && fold(c[k].cp) == ch; };
  while (i < n) {
    size_t j = i;
    // (?i:'s|'t|'re|'ve|'m|'ll|'d)
    if (c[i].cp == '\'') {
      if (isf(i + 1, 's') || isf(i + 1, 't')) j = i + 2;
      else if ((isf(i + 1, 'r') && isf(i + 2, 'e')) || (isf(i + 1, 'v') && isf(i + 2, 'e'))) j = i + 3;
      else if (isf(i + 1, 'm')) j = i + 2;
      else if (isf(i + 1, 'l') && isf(i + 2, 'l')) j = i + 3;
      else if (isf(i + 1, 'd')) j = i + 2;
    }
    // [^\r\n\p{L}\p{N}]?\p{L}+
    if (j == i) {
      size_t s = i;
      if (c[i].cls != kLetter && c[i].cls != kNumber && !is_nl(c[i].cp) && i + 1 < n && c[i + 1].cls == kLetter) s = i + 1;
      if (c[s].cls == kLetter) {
        j = s;
        while (j < n && c[j].cls == kLetter) ++j;
      }
    }
    // \p{N}{1,K}
    if (j == i && c[i].cls == kNumber) {
      j = i;
      while (j < n && c[j].cls == kNumber && j - i < (size_t)K) ++j;
    }
    //  ?[^\s\p{L}\p{N}]+[\r\n]*
    if (j == i) {
      const size_t s = (c[i].cp == ' ' && i + 1 < n && c[i + 1].cls == kOther) ? i + 1 : i;
      if (c[s].cls == kOther) {
        j = s;
        while (j < n && c[j].cls == kOther) ++j;
        while (j < n && is_nl(c[j].cp)) ++j;
      }
    }
    if (j == i) {
      size_t e = i;
      while (e < n && c[e].cls == kSpace) ++e;  // the whole whitespace run
      // \s*[\r\n]+ : up to and including the last CR / LF of the run
      size_t last_nl = n;
      for (size_t k = i; k < e; ++k)
        if (is_nl(c[k].cp)) last_nl = k;
      if (last_nl != n) j = last_nl + 1;
      else if (e == n) j = e;              // \s+(?!\S): the run reaches the end
      else if (e - i >= 2) j = e - 1;      // \s+(?!\S): backtrack one char so that a space follows
      else j = e;                          // \s+
    }
    out->emplace_back(i, j);
    i = j;
  }
}

// The DeepSeek-V3 / R1 pre-tokenizer: Sequence[Split(\p{N}{1,3}), Split([一-龥぀-ゟ゠-ヿ]+), Split(main regex)], every
// Split with behaviour Isolated — matches AND the text between matches become pieces, and the next Split runs inside
// each piece separately (pre_tokenizers/split.rs, pre_tokenizers/sequence.rs).
//   main regex = [!-/:-@\[-`{-~][A-Za-z]+ | [^\r\n\p{L}\p{P}\p{S}]?[\p{L}\p{M}]+ | " ?"[\p{P}\p{S}]+[\r\n]* | \s*[\r\n]+
//                | \s+(?!\S) | \s+          (leftmost-first; a char no alternative matches stays unmatched text)
inline bool ds_cjk(uint32_t cp) {
  return (cp >= 0x4E00 && cp <= 0x9FA5) || (cp >= 0x3040 && cp <= 0x309F) || (cp >= 0x30A0 && cp <= 0x30FF);
}
inline bool ds_ascii_punct(uint32_t cp) {
  return (cp >= 0x21 && cp <= 0x2F) || (cp >= 0x3A && cp <= 0x40) || (cp >= 0x5B && cp <= 0x60) || (cp >= 0x7B && cp <= 0x7E);
}
inline bool ds_ascii_alpha(uint32_t cp) { return (cp >= 'A' && cp <= 'Z') || (cp >= 'a' && cp <= 'z'); }

// one match attempt of the main regex at position i of the piece [b, e); returns the end, or i when nothing matches
size_t ds3_match_at(const std::vector<Ch>& c, const std::vector<int>& sub, size_t i, size_t e) {
  auto is_lm = [&](size_t k) { return c[k].cls == kLetter || (c[k].cls == kOther && sub[k] == kSubM); };
  auto is_ps = [&](size_t k) { return c[k].cls == kOther && (sub[k] == kSubP || sub[k] == kSubS); };
  // [!-/:-@\[-`{-~][A-Za-z]+
  if (ds_ascii_punct(c[i].cp) && i + 1 < e && ds_ascii_alpha(c[i + 1].cp)) {
    size_t j = i + 2;
    while (j < e && ds_ascii_alpha(c[j].cp)) ++j;
    return j;
  }
  // [^\r\n\p{L}\p{P}\p{S}]?[\p{L}\p{M}]+
  {
    size_t s = i;
    if (!is_nl(c[i].cp) && c[i].cls != kLetter && !is_ps(i) && i + 1 < e && is_lm(i + 1)) s = i + 1;
    if (is_lm(s)) {
      size_t j = s;
      while (j < e && is_lm(j)) ++j;
      return j;
    }
  }
  // " ?"[\p{P}\p{S}]+[\r\n]*
  {
    const size_t s = (c[i].cp == ' ' && i + 1 < e && is_ps(i + 1)) ? i + 1 : i;
    if (is_ps(s)) {
      size_t j = s;
      while (j < e && is_ps(j)) ++j;
      while (j < e && is_nl(c[j].cp)) ++j;
      return j;
    }
  }
  if (c[i].cls == kSpace) {
    size_t w = i;
    while (w < e && c[w].cls == kSpace) ++w;  // the whole whitespace run (inside this piece)
    size_t last_nl = e;
    for (size_t k = i; k < w; ++k)
      if (is_nl(c[k].cp)) last_nl = k;
    if (last_nl != e) return last_nl + 1;     // \s*[\r\n]+ : up to and including the last CR / LF of the run
    if (w == e) return w;                     // \s+(?!\S): the run reaches the end of the piece
    if (w - i >= 2) return w - 1;             // \s+(?!\S): backtrack one char so that whitespace follows
    return w;                                 // \s+
  }
  return i;
}

void ds3_split(const std::vector<Ch>& c, std::vector<std::pair<size_t, size_t>>* out) {
  const size_t n = c.size();
  std::vector<int> sub(n);
  for (size_t k = 0; k < n; ++k) sub[k] = uni_sub(c[k].cp);
  size_t i = 0;
  while (i < n) {
    if (c[i].cls == kNumber) {          // stage 1: \p{N}{1,3}, Isolated
      size_t j = i;
      while (j < n && c[j].cls == kNumber && j - i < 3) ++j;
      out->emplace_back(i, j);
      i = j;
      continue;
    }
    if (ds_cjk(c[i].cp)) {              // stage 2: the CJK / kana run, Isolated
      size_t j = i;
      while (j < n && ds_cjk(c[j].cp) && c[j].cls != kNumber) ++j;
      out->emplace_back(i, j);
      i = j;
      continue;
    }
    // stage 3 inside the piece [i, e): up to the next number or CJK char
    size_t e = i;
    while (e < n && c[e].cls != kNumber && !ds_cjk(c[e].cp)) ++e;
    size_t k = i;
    while (k < e) {
      const size_t j = ds3_match_at(c, sub, k, e);
      if (j > k) {
        out->emplace_back(k, j);
        k = j;
      } else {                          // unmatched text up to the next match start = one piece
        size_t u = k + 1;
        while (u < e && ds3_match_at(c, sub, u, e) == u) ++u;
        out->emplace_back(k, u);
        k = u;
      }
    }
    i = e;
  }
}

// models/bpe/word.rs merge_all
struct Sym {
  int32_t id;
  int prev, next;
  bool dead;
};
struct Mg {
  uint32_t rank;
  int pos;
  int32_t new_id;
};
struct MgCmp {
  bool operator()(const Mg& a, const Mg& b) const { return a.rank != b.rank ? a.rank > b.rank : a.pos > b.pos; }
};

void bpe_word(const Hf& h, const uint8_t* bytes, size_t n, std::vector<int32_t>* ids) {
  std::vector<Sym> s(n);
  for (size_t i = 0; i < n; ++i) s[i] = Sym{h.byte_sym[bytes[i]], (int)i - 1, i + 1 < n ? (int)i + 1 : -1, false};
  std::priority_queue<Mg, std::vector<Mg>, MgCmp> q;
  auto push = [&](int pos) {
    if (pos < 0 || s[pos].next < 0) return;
    auto it = h.merges.find(((uint64_t)(uint32_t)s[pos].id << 32) | (uint32_t)s[s[pos].next].id);
    if (it != h.merges.end()) q.push(Mg{it->second.first, pos, it->second.second});
  };
  for (size_t i = 0; i + 1 < n; ++i) push((int)i);
  while (!q.empty()) {
    const Mg top = q.top();
    q.pop();
    if (s[top.pos].dead || s[top.pos].next < 0) continue;
    const int r = s[top.pos].next;
    auto it = h.merges.find(((uint64_t)(uint32_t)s[top.pos].id << 32) | (uint32_t)s[r].id);
    if (it == h.merges.end() || it->second.second != top.new_id) continue;  // expired entry
    s[top.pos].id = top.new_id;
    s[top.pos].next = s[r].next;
    if (s[r].next >= 0) s[s[r].next].prev = top.pos;
    s[r].dead = true;
    push(s[top.pos].prev);
    push(top.pos);
  }
  for (int i = 0; i >= 0 && (size_t)i < n; i = s[i].next) ids->push_back(s[i].id);
}

// leftmost-longest added token of one pass (normalized == which) in text[from, to): its start (to = none)
size_t next_added(const Hf& h, const uint8_t* text, size_t from, size_t to, bool which, size_t* len, int32_t* id) {
  for (size_t p = from; p < to; ++p) {
    size_t best = 0;
    for (size_t a = 0; a < h.added.size(); ++a) {
      const std::string& s = h.added[a].first;
      if (h.added_normalized[a] == which && s.size() <= to - p && s.size() > best && memcmp(text + p, s.data(), s.size()) == 0) {
        best = s.size();
        *id = h.added[a].second;
      }
    }
    if (best) { *len = best; return p; }
  }
  return to;
}

long encode(const Hf& h, const uint8_t* text, size_t len, std::vector<int32_t>* ids) {
  // added_vocabulary.rs extract_and_normalize: split on the non-normalized tokens, then match the normalized ones
  // inside the pieces between them only
  std::vector<std::pair<size_t, size_t>> cut;   // (start, length) of every added token, in text order
  std::vector<int32_t> cut_id;
  for (size_t pos = 0; pos <= len;) {
    size_t l1 = 0, l2 = 0;
    int32_t id1 = -1, id2 = -1;
    const size_t at1 = next_added(h, text, pos, len, false, &l1, &id1);
    for (size_t q = pos; q < at1;) {
      const size_t at2 = next_added(h, text, q, at1, true, &l2, &id2);
      if (at2 == at1) break;
      cut.emplace_back(at2, l2);
      cut_id.push_back(id2);
      q = at2 + l2;
    }
    if (at1 == len) break;
    cut.emplace_back(at1, l1);
    cut_id.push_back(id1);
    pos = at1 + l1;
  }
  size_t pos = 0;
  for (size_t k = 0; k <= cut.size(); ++k) {
    const size_t best_at = k < cut.size() ? cut[k].first : len;
    // ordinary text [pos, best_at)
    std::vector<Ch> c;
    for (size_t p = pos; p < best_at;) {
      uint32_t cp;
      const int l = decode(text + p, best_at - p, &cp);
      if (l == 0) return -1;  // malformed UTF-8: the Rust shim panics
      c.push_back(Ch{cp, uni_class(cp), (uint32_t)p, (uint32_t)l});
      p += l;
    }
    std::vector<std::pair<size_t, size_t>> pieces;
    if (h.pattern == 3) ds3_split(c, &pieces);
    else if (h.pattern == 2) cl100k_split(c, h.digits, &pieces);
    else gpt2_split(c, &pieces);
    for (const auto& pr : pieces) {
      const size_t b = c[pr.first].off, e = c[pr.second - 1].off + c[pr.second - 1].len;
      if (h.ignore_merges) {
        auto it = h.vocab.find(std::string((const char*)text + b, e - b));
        if (it != h.vocab.end()) { ids->push_back(it->second); continue; }
      }
      bpe_word(h, text + b, e - b, ids);
    }
    if (k == cut.size()) break;
    ids->push_back(cut_id[k]);
    pos = best_at + cut[k].second;
  }
  return (long)ids->size();
}

}  // namespace

extern "C" {

// byte_sym[256]: id of each byte's byte-level char; merges: n x (left id, right id, new id), rank = index;
// added: n_added strings (blob + offsets) with their ids and `normalized` flags (null: none normalized).
void* oracle_hf_new(const int32_t* byte_sym, const int32_t* merges, size_t n_merges, const char* added_blob,
                    const int64_t* added_off, const int32_t* added_ids, const uint8_t* added_normalized, size_t n_added) {
  Hf* h = new Hf();
  memcpy(h->byte_sym, byte_sym, sizeof(h->byte_sym));
  for (size_t i = 0; i < n_merges; ++i)
    h->merges.emplace(((uint64_t)(uint32_t)merges[3 * i] << 32) | (uint32_t)merges[3 * i + 1],
                      std::make_pair((uint32_t)i, merges[3 * i + 2]));
  for (size_t i = 0; i < n_added; ++i) {
    h->added.emplace_back(std::string(added_blob + added_off[i], (size_t)(added_off[i + 1] - added_off[i])), added_ids[i]);
    h->added_normalized.push_back(added_normalized && added_normalized[i]);
  }
  return h;
}
// pattern: 1 GPT-2 / 2 cl100k family (digits = K) / 3 DeepSeek-V3 three-stage split; vocab: raw bytes of every token (blob + offsets) with ids,
// consulted per pre-token when ignore_merges is set
void oracle_hf_configure(void* hv, int pattern, int digits, int ignore_merges, const char* vocab_blob,
                         const int64_t* vocab_off, const int32_t* vocab_ids, size_t n_vocab) {
  Hf* h = (Hf*)hv;
  h->pattern = pattern;
  h->digits = digits;
  h->ignore_merges = ignore_merges != 0;
  h->vocab.clear();
  for (size_t i = 0; i < n_vocab; ++i)
    h->vocab.emplace(std::string(vocab_blob + vocab_off[i], (size_t)(vocab_off[i + 1] - vocab_off[i])), vocab_ids[i]);
}
void oracle_hf_free(void* h) { delete (Hf*)h; }
// FastTokenizer::encode; returns the id count, or -1 for malformed UTF-8 (the reference aborts there).
long oracle_hf_encode(void* h, const char* text, size_t len, int32_t* out, size_t cap) {
  std::vector<int32_t> ids;
  const long n = encode(*(Hf*)h, (const uint8_t*)text, len, &ids);
  if (n < 0) return -1;
  memcpy(out, ids.data(), sizeof(int32_t) * (ids.size() < cap ? ids.size() : cap));
  return n;
}

}  // extern "C"
