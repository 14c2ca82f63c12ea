// oracle/sp_oracle.cc -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// CPU restatement of the tokenize step of the reference's ingest path for the
// SentencePiece backend:
//   xllm_service/tokenizer/sentencepiece_tokenizer.cpp:47-50   sp_processor_.Load(<dir>/tokenizer.model)
//   xllm_service/tokenizer/sentencepiece_tokenizer.cpp:115-128 encode_internal: empty text -> true;
//        sp_processor_.Encode(text, &spt); ids = spt.pieces[i].id
//   xllm_service/tokenizer/sentencepiece_tokenizer.cpp:130-168 encode: prefix tokens / special-token
//        regex are never configured by the service (tokenizer_args.cpp:30-71), so encode ==
//        encode_internal(text) APPENDING to *ids.
//
// All arithmetic lives in the third-party library the reference links:
//   sentencepiece @ ca10c9975797a4979b3c9fde33a14b2f92d1961d (third_party/sentencepiece, absent
//   from the reference checkout).  This file restates its published algorithm for BPE models:
//     normalizer.cc  Normalizer::Normalize / NormalizePrefix (precompiled charsmap = Darts
//                    double-array trie + replacement blob; whitespace rules)
//     bpe_model.cc   Model::Encode (agenda of adjacent symbol pairs: highest score first,
//                    leftmost on ties; stale-entry check by merged size)
//     sentencepiece_processor.cc  PopulateSentencePieceText (byte fallback; merging of
//                    consecutive unknown pieces when byte fallback is off)
//     model_interface.cc  InitializePieces / PieceToId (reserved map first)
//   It is pinned against upstream libsentencepiece (pip sentencepiece 0.2.1) by
//   tests/test_oracle_sp.py: live when the wheel is importable, and through the committed
//   vectors tests/golden/sp_bpe_8k_goldens.json.
//
//     unigram_model.cc  Model::EncodeOptimized (UNIGRAM models: Viterbi over the normalized bytes, on-the-fly
//                    lattice; candidate scores are formed in double and stored as float, the earlier / shorter
//                    candidate wins ties, a char no piece covers costs min_score - 10)
//     model_interface.cc / normalizer.cc / bpe_model.cc  USER_DEFINED pieces: matched longest-first on the raw
//                    text (PrefixMatcher), copied through the normalizer verbatim, never merged (BPE: frozen
//                    symbols) / always preferred (Unigram: score = length * max_score - 0.1)
// Unsupported (load fails): WORD/CHAR models, UNUSED pieces.
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <queue>
#include <string>
#include <string_view>
#include <thread>
#include <unordered_map>
#include <vector>

namespace {

// ---------------------------------------------------------------- protobuf wire reader
struct PbReader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  PbReader(const void* d, size_t n) : p((const uint8_t*)d), end((const uint8_t*)d + n) {}
  bool done() const { return p >= end || !ok; }
  uint64_t varint() {
    uint64_t v = 0;
    int shift = 0;
    while (p < end && shift < 64) {
      uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
      shift += 7;
    }
    ok = false;
    return 0;
  }
  // returns field number, sets wire type; for len-delimited sets (data,len)
  bool next(uint32_t* field, uint32_t* wt, uint64_t* val, std::string_view* bytes) {
    if (done()) return false;
    uint64_t key = varint();
    if (!ok) return false;
    *field = (uint32_t)(key >> 3);
    *wt = (uint32_t)(key & 7);
    switch (*wt) {
      case 0: *val = varint(); return ok;
      case 1:
        if (end - p < 8) { ok = false; return false; }
        memcpy(val, p, 8); p += 8; return true;
      case 2: {
        uint64_t n = varint();
        if (!ok || (uint64_t)(end - p) < n) { ok = false; return false; }
        *bytes = std::string_view((const char*)p, (size_t)n);
        p += n;
        return true;
      }
      case 5: {
        if (end - p < 4) { ok = false; return false; }
        uint32_t v32; memcpy(&v32, p, 4); p += 4; *val = v32; return true;
      }
      default: ok = false; return false;
    }
  }
};

enum PieceType { NORMAL = 1, UNKNOWN = 2, CONTROL = 3, USER_DEFINED = 4, UNUSED = 5, BYTE = 6 };

struct Piece {
  std::string piece;
  float score = 0.f;
  int type = NORMAL;
};

struct SpModel {
  std::vector<Piece> pieces;
  int model_type = 1;  // TrainerSpec.model_type default UNIGRAM
  bool byte_fallback = false;
  bool treat_whitespace_as_suffix = false;
  int unk_id = -1;
  // normalizer spec
  std::string charsmap;
  bool add_dummy_prefix = true;
  bool remove_extra_whitespaces = true;
  bool escape_whitespaces = true;
  // derived
  const uint32_t* trie = nullptr;
  size_t trie_units = 0;
  const char* norm_blob = nullptr;
  size_t norm_blob_size = 0;
  std::unordered_map<std::string_view, int> pieces_map;    // NORMAL / USER_DEFINED / UNUSED
  std::unordered_map<std::string_view, int> reserved_map;  // CONTROL / UNKNOWN / BYTE
  int byte_id[256];
  // unigram_model.cc: min / max over NORMAL pieces, longest piece in bytes
  float min_score = 0.f, max_score = 0.f;
  size_t max_piece_len = 0;
  std::vector<std::string_view> user_defined;  // model_interface.cc: the PrefixMatcher's symbols
  std::string error;
};

bool parse_model(const std::string& blob, SpModel* m) {
  PbReader r(blob.data(), blob.size());
  uint32_t f, wt; uint64_t v; std::string_view b;
  while (r.next(&f, &wt, &v, &b)) {
    if (f == 1 && wt == 2) {  // repeated SentencePiece pieces
      Piece pc;
      PbReader pr(b.data(), b.size());
      uint32_t pf, pwt; uint64_t pv; std::string_view pb;
      while (pr.next(&pf, &pwt, &pv, &pb)) {
        if (pf == 1 && pwt == 2) pc.piece.assign(pb.data(), pb.size());
        else if (pf == 2 && pwt == 5) { uint32_t u = (uint32_t)pv; memcpy(&pc.score, &u, 4); }
        else if (pf == 3 && pwt == 0) pc.type = (int)pv;
      }
      if (!pr.ok) { m->error = "bad SentencePiece message"; return false; }
      m->pieces.push_back(std::move(pc));
    } else if (f == 2 && wt == 2) {  // TrainerSpec
      PbReader tr(b.data(), b.size());
      uint32_t tf, twt; uint64_t tv; std::string_view tb;
      while (tr.next(&tf, &twt, &tv, &tb)) {
        if (tf == 3 && twt == 0) m->model_type = (int)tv;
        else if (tf == 35 && twt == 0) m->byte_fallback = tv != 0;
        else if (tf == 24 && twt == 0) m->treat_whitespace_as_suffix = tv != 0;
      }
      if (!tr.ok) { m->error = "bad TrainerSpec"; return false; }
    } else if (f == 3 && wt == 2) {  // NormalizerSpec
      PbReader nr(b.data(), b.size());
      uint32_t nf, nwt; uint64_t nv; std::string_view nb;
      while (nr.next(&nf, &nwt, &nv, &nb)) {
        if (nf == 2 && nwt == 2) m->charsmap.assign(nb.data(), nb.size());
        else if (nf == 3 && nwt == 0) m->add_dummy_prefix = nv != 0;
        else if (nf == 4 && nwt == 0) m->remove_extra_whitespaces = nv != 0;
        else if (nf == 5 && nwt == 0) m->escape_whitespaces = nv != 0;
      }
      if (!nr.ok) { m->error = "bad NormalizerSpec"; return false; }
    }
  }
  if (!r.ok) { m->error = "bad ModelProto"; return false; }
  return true;
}

// model_interface.cc InitializePieces
bool init_pieces(SpModel* m) {
  for (int i = 0; i < 256; ++i) m->byte_id[i] = -1;
  for (size_t i = 0; i < m->pieces.size(); ++i) {
    const Piece& sp = m->pieces[i];
    if (sp.piece.empty()) { m->error = "piece must not be empty."; return false; }
    const bool is_normal = sp.type == NORMAL || sp.type == USER_DEFINED || sp.type == UNUSED;
    auto& map = is_normal ? m->pieces_map : m->reserved_map;
    if (!map.emplace(std::string_view(sp.piece), (int)i).second) {
      m->error = sp.piece + " is already defined.";
      return false;
    }
    if (sp.type == UNUSED) {
      m->error = "UNUSED pieces are not supported by this oracle";
      return false;
    }
    if (sp.type == USER_DEFINED) m->user_defined.push_back(std::string_view(sp.piece));
    if (sp.type == UNKNOWN) {
      if (m->unk_id >= 0) { m->error = "unk is already defined."; return false; }
      m->unk_id = (int)i;
    }
    if (sp.type == BYTE) {
      if (!m->byte_fallback) { m->error = "byte piece is found although `byte_fallback` is false."; return false; }
      unsigned int bv = 0;
      if (sp.piece.size() != 6 || sscanf(sp.piece.c_str(), "<0x%02X>", &bv) != 1) {
        m->error = "byte piece " + sp.piece + " is invalid.";
        return false;
      }
      m->byte_id[bv & 0xFF] = (int)i;
    }
  }
  if (m->unk_id < 0) { m->error = "unk is not defined."; return false; }
  {  // unigram_model.cc Model::PopulateNodes / constructor: score range over the NORMAL pieces
    float mn = 3.402823466e+38f, mx = 1.175494351e-38f;  // FLT_MAX, FLT_MIN as upstream initialises them
    for (const Piece& sp : m->pieces) {
      if (sp.type == NORMAL) {
        mn = sp.score < mn ? sp.score : mn;
        mx = sp.score > mx ? sp.score : mx;
      }
      if ((sp.type == NORMAL || sp.type == USER_DEFINED) && sp.piece.size() > m->max_piece_len)
        m->max_piece_len = sp.piece.size();
    }
    m->min_score = mn;
    m->max_score = mx;
  }
  if (m->byte_fallback)
    for (int i = 0; i < 256; ++i)
      if (m->byte_id[i] < 0) { m->error = "there are not 256 byte pieces although `byte_fallback` is true."; return false; }
  // normalizer.cc DecodePrecompiledCharsMap
  if (!m->charsmap.empty()) {
    uint32_t trie_size = 0;
    if (m->charsmap.size() <= 4) { m->error = "Blob for normalization rule is broken."; return false; }
    memcpy(&trie_size, m->charsmap.data(), 4);
    if (trie_size >= m->charsmap.size() || trie_size % 4 != 0) { m->error = "Trie data size exceeds the input blob size."; return false; }
    m->trie = reinterpret_cast<const uint32_t*>(m->charsmap.data() + 4);
    m->trie_units = trie_size / 4;
    m->norm_blob = m->charsmap.data() + 4 + trie_size;
    m->norm_blob_size = m->charsmap.size() - 4 - trie_size;
  }
  return true;
}

// ---------------------------------------------------------------- UTF-8 (util.cc)
inline bool is_trail(uint8_t x) { return (int8_t)x < -0x40; }
inline bool is_valid_cp(uint32_t c) { return c < 0xD800 || (c >= 0xE000 && c <= 0x10FFFF); }
constexpr uint32_t kUnicodeError = 0xFFFD;

uint32_t decode_utf8(const uint8_t* b, const uint8_t* e, size_t* mblen) {
  const size_t len = e - b;
  if (b[0] < 0x80) { *mblen = 1; return b[0]; }
  if (len >= 2 && (b[0] & 0xE0) == 0xC0) {
    const uint32_t cp = ((b[0] & 0x1F) << 6) | (b[1] & 0x3F);
    if (is_trail(b[1]) && cp >= 0x0080 && is_valid_cp(cp)) { *mblen = 2; return cp; }
  } else if (len >= 3 && (b[0] & 0xF0) == 0xE0) {
    const uint32_t cp = ((b[0] & 0x0F) << 12) | ((b[1] & 0x3F) << 6) | (b[2] & 0x3F);
    if (is_trail(b[1]) && is_trail(b[2]) && cp >= 0x0800 && is_valid_cp(cp)) { *mblen = 3; return cp; }
  } else if (len >= 4 && (b[0] & 0xF8) == 0xF0) {
    const uint32_t cp = ((b[0] & 0x07) << 18) | ((b[1] & 0x3F) << 12) | ((b[2] & 0x3F) << 6) | (b[3] & 0x3F);
    if (is_trail(b[1]) && is_trail(b[2]) && is_trail(b[3]) && cp >= 0x10000 && is_valid_cp(cp)) { *mblen = 4; return cp; }
  }
  *mblen = 1;
  return kUnicodeError;
}
inline bool is_valid_decode_utf8(const uint8_t* b, const uint8_t* e, size_t* mblen) {
  const uint32_t c = decode_utf8(b, e, mblen);
  return c != kUnicodeError || *mblen == 3;
}
inline size_t one_char_len(const char* s) { return "\1\1\1\1\1\1\1\1\1\1\1\1\2\2\3\4"[(*(const uint8_t*)s & 0xFF) >> 4]; }

// ---------------------------------------------------------------- normalizer.cc
// Darts-clone double-array unit accessors.
inline bool da_has_leaf(uint32_t u) { return ((u >> 8) & 1) == 1; }
inline uint32_t da_value(uint32_t u) { return u & ((1U << 31) - 1); }
inline uint32_t da_label(uint32_t u) { return u & ((1U << 31) | 0xFF); }
inline uint32_t da_offset(uint32_t u) { return (u >> 10) << ((u & (1U << 9)) >> 6); }

// normalizer.cc PrefixMatcher::PrefixMatch: the longest user-defined symbol that is a prefix of w (0 = none)
inline size_t user_prefix_match(const SpModel& m, const char* w, size_t len) {
  size_t best = 0;
  for (std::string_view u : m.user_defined)
    if (u.size() > best && u.size() <= len && memcmp(w, u.data(), u.size()) == 0) best = u.size();
  return best;
}

// NormalizePrefix: returns (replacement, consumed bytes)
inline std::pair<std::string_view, int> normalize_prefix(const SpModel& m, const char* in, size_t len) {
  if (len == 0) return {std::string_view(), 0};
  if (!m.user_defined.empty()) {  // user-defined symbols pass through verbatim
    const size_t u = user_prefix_match(m, in, len);
    if (u) return {std::string_view(in, u), (int)u};
  }
  size_t longest_length = 0;
  int longest_value = 0;
  if (m.trie) {
    // commonPrefixSearch; upstream keeps at most 32 results and takes the longest among them.
    size_t num = 0;
    uint32_t node = 0;
    uint32_t unit = m.trie[node];
    node ^= da_offset(unit);
    for (size_t i = 0; i < len; ++i) {
      node ^= (uint8_t)in[i];
      if (node >= m.trie_units) break;
      unit = m.trie[node];
      if (da_label(unit) != (uint8_t)in[i]) break;
      node ^= da_offset(unit);
      if (da_has_leaf(unit)) {
        if (num < 32) {
          const size_t l = i + 1;
          if (longest_length == 0 || l > longest_length) {
            longest_length = l;
            longest_value = (int)da_value(m.trie[node]);
          }
        }
        ++num;
      }
    }
  }
  if (longest_length == 0) {
    size_t length = 0;
    if (!is_valid_decode_utf8((const uint8_t*)in, (const uint8_t*)in + len, &length)) {
      return {std::string_view("\xEF\xBF\xBD", 3), 1};
    }
    return {std::string_view(in, length), (int)length};
  }
  return {std::string_view(m.norm_blob + longest_value), (int)longest_length};  // NUL-delimited
}

void normalize(const SpModel& m, std::string_view input, std::string* out) {
  out->clear();
  if (input.empty()) return;
  const char* in = input.data();
  size_t len = input.size();
  if (m.remove_extra_whitespaces) {
    while (len > 0) {
      auto p = normalize_prefix(m, in, len);
      if (p.first != " ") break;
      in += p.second;
      len -= p.second;
    }
  }
  if (len == 0) return;
  out->reserve(len * 3);
  static const char kSpace[] = "\xe2\x96\x81";
  auto add_ws = [&]() {
    if (m.escape_whitespaces) out->append(kSpace, 3);
    else out->push_back(' ');
  };
  if (!m.treat_whitespace_as_suffix && m.add_dummy_prefix) add_ws();
  bool is_prev_space = m.remove_extra_whitespaces;
  while (len > 0) {
    auto p = normalize_prefix(m, in, len);
    std::string_view sp = p.first;
    while (is_prev_space && !sp.empty() && sp[0] == ' ') sp.remove_prefix(1);
    if (!sp.empty()) {
      for (char c : sp) {
        if (m.escape_whitespaces && c == ' ') out->append(kSpace, 3);
        else out->push_back(c);
      }
      is_prev_space = sp.back() == ' ';
    }
    in += p.second;
    len -= p.second;
    if (!m.remove_extra_whitespaces) is_prev_space = false;
  }
  if (m.remove_extra_whitespaces) {
    const std::string_view space = m.escape_whitespaces ? std::string_view(kSpace, 3) : std::string_view(" ");
    while (out->size() >= space.size() && out->compare(out->size() - space.size(), space.size(), space) == 0)
      out->resize(out->size() - space.size());
  }
  if (m.treat_whitespace_as_suffix && m.add_dummy_prefix) add_ws();
}

// ---------------------------------------------------------------- bpe_model.cc Model::Encode
struct SymbolPair {
  int left, right;
  float score;
  size_t size;
};
struct PairCmp {
  bool operator()(const SymbolPair& a, const SymbolPair& b) const {
    return a.score < b.score || (a.score == b.score && a.left > b.left);
  }
};
struct Symbol {
  bool freeze = false;  // a user-defined symbol: never merged
  int prev, next;
  std::string_view piece;
};

inline int piece_to_id(const SpModel& m, std::string_view w) {
  auto it = m.reserved_map.find(w);
  if (it != m.reserved_map.end()) return it->second;
  auto it2 = m.pieces_map.find(w);
  if (it2 != m.pieces_map.end()) return it2->second;
  return m.unk_id;
}

struct EncodeScratch {
  std::string normalized;
  std::vector<Symbol> symbols;
  std::vector<SymbolPair> heap;
};

// sentencepiece_processor.cc PopulateSentencePieceText for one (piece, id): byte fallback, merging of
// consecutive unknown pieces when byte fallback is off
inline void emit_piece(const SpModel& m, std::string_view w, int id, bool* is_prev_unk, std::vector<int32_t>* ids) {
  const bool is_unk = m.pieces[id].type == UNKNOWN;
  if (m.pieces[id].type == CONTROL) {
    ids->push_back(id);
  } else if (is_unk && m.byte_fallback) {
    for (char c : w) ids->push_back(m.byte_id[(uint8_t)c]);
  } else if (*is_prev_unk && is_unk) {
    // consecutive unknown pieces are merged into the previous piece: no new id
  } else {
    ids->push_back(id);
  }
  *is_prev_unk = is_unk;
}

// unigram_model.cc Model::EncodeOptimized
void encode_unigram(const SpModel& m, std::string_view normalized, std::vector<int32_t>* ids) {
  struct Node {
    int id = -1;
    float best = 0.f;
    int starts_at = -1;
  };
  const int size = (int)normalized.size();
  const float unk_score = m.min_score - 10.0f;  // kUnkPenalty
  std::vector<Node> ends_at((size_t)size + 1);
  int starts_at = 0;
  while (starts_at < size) {
    const float till_here = ends_at[(size_t)starts_at].best;
    bool has_single_node = false;
    const int mblen = std::min<int>((int)one_char_len(normalized.data() + starts_at), size - starts_at);
    // every piece that is a prefix of the rest, shortest first (the order the trie walk meets them)
    const int max_len = std::min<int>((int)m.max_piece_len, size - starts_at);
    for (int len = 1; len <= max_len; ++len) {
      auto it = m.pieces_map.find(normalized.substr((size_t)starts_at, (size_t)len));
      if (it == m.pieces_map.end()) continue;
      Node& t = ends_at[(size_t)(starts_at + len)];
      // `auto score = user_defined ? (length * max_score_ - 0.1) : GetScore(id)` upstream: a double either way
      const double score = m.pieces[(size_t)it->second].type == USER_DEFINED
                               ? (double)((float)len * m.max_score) - 0.1
                               : (double)m.pieces[(size_t)it->second].score;
      const double cand = score + (double)till_here;
      if (t.starts_at == -1 || cand > (double)t.best) {
        t.best = (float)cand;
        t.starts_at = starts_at;
        t.id = it->second;
      }
      if (!has_single_node && len == mblen) has_single_node = true;
    }
    if (!has_single_node) {
      Node& t = ends_at[(size_t)(starts_at + mblen)];
      const float cand = unk_score + till_here;  // both float upstream
      if (t.starts_at == -1 || cand > t.best) {
        t.best = cand;
        t.starts_at = starts_at;
        t.id = m.unk_id;
      }
    }
    starts_at += mblen;
  }
  std::vector<std::pair<int, int>> path;  // (start, end) backwards
  for (int e = size; e > 0;) {
    const Node& nd = ends_at[(size_t)e];
    path.emplace_back(nd.starts_at, e);
    e = nd.starts_at;
  }
  bool is_prev_unk = false;
  for (size_t i = path.size(); i-- > 0;) {
    const int b = path[i].first, e = path[i].second;
    emit_piece(m, normalized.substr((size_t)b, (size_t)(e - b)), ends_at[(size_t)e].id, &is_prev_unk, ids);
  }
}

// SentencePieceProcessor::Encode -> ids appended to *ids.
void encode(const SpModel& m, std::string_view text, EncodeScratch* sc, std::vector<int32_t>* ids) {
  if (text.empty()) return;  // sentencepiece_tokenizer.cpp:117-120
  normalize(m, text, &sc->normalized);
  std::string_view normalized(sc->normalized);
  if (normalized.empty()) return;
  if (m.model_type == 1) { encode_unigram(m, normalized, ids); return; }
  auto& symbols = sc->symbols;
  symbols.clear();
  std::priority_queue<SymbolPair, std::vector<SymbolPair>, PairCmp> agenda(PairCmp(), std::move(sc->heap));
  auto maybe_add = [&](int left, int right) {
    if (left == -1 || right == -1 || symbols[left].freeze || symbols[right].freeze) return;
    const std::string_view piece(symbols[left].piece.data(), symbols[left].piece.size() + symbols[right].piece.size());
    auto it = m.pieces_map.find(piece);
    if (it == m.pieces_map.end()) return;
    agenda.push(SymbolPair{left, right, m.pieces[it->second].score, piece.size()});
  };
  {
    int index = 0;
    std::string_view rest = normalized;
    while (!rest.empty()) {
      Symbol s;
      const size_t ulen = m.user_defined.empty() ? 0 : user_prefix_match(m, rest.data(), rest.size());
      s.freeze = ulen != 0;
      const size_t mblen = ulen ? ulen : std::min(rest.size(), one_char_len(rest.data()));
      s.piece = std::string_view(rest.data(), mblen);
      s.prev = index == 0 ? -1 : index - 1;
      rest.remove_prefix(mblen);
      s.next = rest.empty() ? -1 : index + 1;
      ++index;
      symbols.push_back(s);
    }
  }
  for (size_t i = 1; i < symbols.size(); ++i) maybe_add((int)i - 1, (int)i);
  while (!agenda.empty()) {
    const SymbolPair top = agenda.top();
    agenda.pop();
    if (symbols[top.left].piece.empty() || symbols[top.right].piece.empty() ||
        symbols[top.left].piece.size() + symbols[top.right].piece.size() != top.size)
      continue;
    symbols[top.left].piece =
        std::string_view(symbols[top.left].piece.data(), symbols[top.left].piece.size() + symbols[top.right].piece.size());
    symbols[top.left].next = symbols[top.right].next;
    if (symbols[top.right].next >= 0) symbols[symbols[top.right].next].prev = top.left;
    symbols[top.right].piece = std::string_view("");
    maybe_add(symbols[top.left].prev, top.left);
    maybe_add(top.left, symbols[top.left].next);
  }
  // PopulateSentencePieceText
  bool is_prev_unk = false;
  for (int index = 0; index != -1; index = symbols[index].next) {
    const std::string_view w = symbols[index].piece;
    emit_piece(m, w, piece_to_id(m, w), &is_prev_unk, ids);
  }
}

struct SpHandle {
  SpModel m;
};

}  // namespace

extern "C" {

// Loads <path> (a tokenizer.model file).  Returns NULL on failure (err gets the message).
void* oracle_sp_load(const char* path, char* err, size_t err_cap) {
  FILE* f = fopen(path, "rb");
  if (!f) {
    if (err) snprintf(err, err_cap, "cannot open %s", path);
    return nullptr;
  }
  std::string blob;
  char buf[1 << 16];
  size_t n;
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) blob.append(buf, n);
  fclose(f);
  SpHandle* h = new SpHandle();
  if (!parse_model(blob, &h->m) || !init_pieces(&h->m)) {
    if (err) snprintf(err, err_cap, "%s", h->m.error.c_str());
    delete h;
    return nullptr;
  }
  if (h->m.model_type != 2 && h->m.model_type != 1) {
    if (err) snprintf(err, err_cap, "model_type %d is neither UNIGRAM (1) nor BPE (2)", h->m.model_type);
    delete h;
    return nullptr;
  }
  return h;
}
void oracle_sp_free(void* h) { delete (SpHandle*)h; }
int oracle_sp_model_type(void* h) { return ((SpHandle*)h)->m.model_type; }  // 1 UNIGRAM, 2 BPE
int oracle_sp_piece_count(void* h) { return (int)((SpHandle*)h)->m.pieces.size(); }

// Normalizer::Normalize.  Returns the normalized length (bytes), writes up to cap bytes.
long oracle_sp_normalize(void* h, const char* text, size_t len, char* out, size_t cap) {
  std::string norm;
  normalize(((SpHandle*)h)->m, std::string_view(text, len), &norm);
  memcpy(out, norm.data(), std::min(cap, norm.size()));
  return (long)norm.size();
}

// SentencePieceTokenizer::encode for one text.  Returns the number of ids (may exceed cap; only cap are written).
long oracle_sp_encode(void* h, const char* text, size_t len, int32_t* ids_out, size_t cap) {
  EncodeScratch sc;
  std::vector<int32_t> ids;
  encode(((SpHandle*)h)->m, std::string_view(text, len), &sc, &ids);
  memcpy(ids_out, ids.data(), sizeof(int32_t) * std::min(cap, ids.size()));
  return (long)ids.size();
}

// Batch over a CSR text buffer with n_threads worker threads, one request at a time per
// thread (the reference's per-request, per-thread model: scheduler.cpp:128-133,274-277).
// ids of request r are written at ids_out + r * ids_stride (truncated to ids_stride), n_ids[r] = count.
// Returns 0.
int oracle_sp_encode_batch(void* h, const char* text, const int64_t* offsets, size_t n_req, int32_t* ids_out,
                           int64_t ids_stride, int32_t* n_ids, int n_threads) {
  const SpModel& m = ((SpHandle*)h)->m;
  std::atomic<size_t> next{0};
  auto work = [&]() {
    EncodeScratch sc;
    std::vector<int32_t> ids;
    for (;;) {
      const size_t r = next.fetch_add(1);
      if (r >= n_req) break;
      ids.clear();
      encode(m, std::string_view(text + offsets[r], (size_t)(offsets[r + 1] - offsets[r])), &sc, &ids);
      n_ids[r] = (int32_t)ids.size();
      memcpy(ids_out + r * ids_stride, ids.data(), sizeof(int32_t) * std::min<size_t>(ids.size(), (size_t)ids_stride));
    }
  };
  if (n_threads <= 1) {
    work();
  } else {
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; ++t) th.emplace_back(work);
    for (auto& t : th) t.join();
  }
  return 0;
}

}  // extern "C"
