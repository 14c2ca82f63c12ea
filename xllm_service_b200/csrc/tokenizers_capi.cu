// tokenizers_capi.cu — the legacy `tokenizers_*` C-ABI (include/tokenizers.h) on top of the batch API.
// Replaces the Rust shim xllm_service/tokenizer/tokenizers/src/lib.rs:56-204 behind the unchanged
// xllm_service/tokenizer/fast_tokenizer.cpp.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/tokenizers.h"
#include "../../include/xllm_ingest.h"
#include "handle.h"

namespace {

struct LegacyTokenizer {
  xllm_ingest_t h = nullptr;
  std::string scratch;  // backs tokenizers_decode / tokenizers_id_to_token results
  std::unordered_map<std::string, int32_t> piece_to_id;
  std::string tmp_model_path;
};

// String::from_utf8_lossy: every maximal subpart of an ill-formed sequence becomes one U+FFFD
std::string utf8_lossy(const std::string& in) {
  const uint8_t* p = (const uint8_t*)in.data();
  const size_t n = in.size();
  std::string out;
  out.reserve(n);
  size_t i = 0;
  while (i < n) {
    const uint8_t b = p[i];
    int len = 0;
    uint8_t lo = 0x80, hi = 0xBF;   // range of the second byte
    if (b < 0x80) len = 1;
    else if (b >= 0xC2 && b <= 0xDF) len = 2;
    else if (b >= 0xE0 && b <= 0xEF) { len = 3; lo = b == 0xE0 ? 0xA0 : 0x80; hi = b == 0xED ? 0x9F : 0xBF; }
    else if (b >= 0xF0 && b <= 0xF4) { len = 4; lo = b == 0xF0 ? 0x90 : 0x80; hi = b == 0xF4 ? 0x8F : 0xBF; }
    size_t k = 1;
    while (len > 1 && (int)k < len && i + k < n && p[i + k] >= (k == 1 ? lo : 0x80) && p[i + k] <= (k == 1 ? hi : 0xBF)) ++k;
    if (len > 0 && (int)k == len) out.append(in, i, (size_t)len);
    else out += "\xEF\xBF\xBD";
    i += len > 0 ? k : 1;
  }
  return out;
}

// SentencePieceProcessor::Decode for BPE pieces: U+2581 -> ' ', byte pieces -> raw bytes, control pieces
// dropped, unknown -> " \xE2\x81\x87 " (the default unk_surface), leading space of the dummy prefix removed.
std::string decode_ids(const xllm::SpTables& t, const uint32_t* ids, size_t n, bool skip_special) {
  std::string out;
  bool first = true;
  for (size_t i = 0; i < n; ++i) {
    if (ids[i] >= t.piece_str.size()) continue;
    const std::string& p = t.piece_str[ids[i]];
    if (t.byte_mode) {
      // tiktoken: tokens are raw byte strings (tiktoken_tokenizer.cpp:296-316); HF byte-level: the ByteLevel
      // decoder maps the vocab spelling back to bytes, special tokens dropped on request (lib.rs:101-113), and the
      // joined bytes read as String::from_utf8_lossy does
      if (!t.piece_raw.empty()) {
        if (!(skip_special && t.piece_type[ids[i]] == 3)) out += t.piece_raw[ids[i]];
      } else {
        out += p;
      }
      continue;
    }
    const int type = t.piece_type[ids[i]];
    if (type == 3) {  // CONTROL
      if (!skip_special) out += p;
      continue;
    }
    if (type == 2) { out += " \xE2\x81\x87 "; first = false; continue; }
    if (type == 6) {  // BYTE: "<0xAB>"
      unsigned v = 0;
      sscanf(p.c_str(), "<0x%02X>", &v);
      out.push_back((char)v);
      first = false;
      continue;
    }
    size_t k = 0;
    while (k < p.size()) {
      if (p.compare(k, 3, "\xE2\x96\x81") == 0) {
        if (!(first && k == 0 && t.add_dummy_prefix)) out.push_back(' ');
        k += 3;
      } else {
        out.push_back(p[k++]);
      }
    }
    first = false;
  }
  return t.byte_mode && !t.piece_raw.empty() ? utf8_lossy(out) : out;
}

LegacyTokenizer* make(const char* path) {
  xllm_ingest_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.tokenizer_path = path;
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess) cfg.device = dev;
  LegacyTokenizer* L = new LegacyTokenizer();
  if (xllm_ingest_create(&cfg, &L->h) != XLLM_OK) {
    delete L;
    return nullptr;
  }
  const xllm::SpTables& t = *L->h->sp_tables;
  for (uint32_t i = 0; i < t.piece_str.size(); ++i)
    if (!t.piece_str[i].empty()) L->piece_to_id.emplace(t.piece_str[i], (int32_t)i);
  return L;
}

// add_special: Tokenizer::encode(text, add_special_tokens) (lib.rs:83-99) — with 0 the template ids a
// tokenizer.json wraps around the sequence are left off (the device always writes them: the service passes 1)
void encode_many(LegacyTokenizer* L, const char* const* data, const size_t* len, size_t n, bool add_special,
                 TokenizerEncodeResult* results) {
  for (size_t i = 0; i < n; ++i) { results[i].token_ids = nullptr; results[i].len = 0; }
  if (!L || n == 0) return;
  std::vector<int64_t> off(n + 1, 0);
  for (size_t i = 0; i < n; ++i) off[i + 1] = off[i] + (int64_t)len[i];
  std::string text;
  text.reserve((size_t)off[n]);
  size_t longest = 0;
  for (size_t i = 0; i < n; ++i) { text.append(data[i], len[i]); longest = len[i] > longest ? len[i] : longest; }
  int64_t stride = (int64_t)longest + 8;  // >= 1 byte per token on ordinary text; grown on truncation
  std::vector<int32_t> ids, n_ids(n), status(n);
  for (int attempt = 0; attempt < 3; ++attempt) {
    ids.assign(n * (size_t)stride, 0);
    if (xllm_encode_batch(L->h, (int32_t)n, reinterpret_cast<const uint8_t*>(text.data()), off.data(), ids.data(),
                          stride, n_ids.data(), status.data()) != XLLM_OK)
      return;
    int64_t need = 0;
    for (size_t i = 0; i < n; ++i)
      if (status[i] == XLLM_ENC_TRUNCATED && n_ids[i] > need) need = n_ids[i];
    if (!need) break;
    stride = need;
  }
  const xllm::SpTables& t = *L->h->sp_tables;
  const size_t cut_front = add_special ? 0 : t.prefix_ids.size(), cut_back = add_special ? 0 : t.suffix_ids.size();
  for (size_t i = 0; i < n; ++i) {
    if (status[i] != XLLM_OK) continue;
    const size_t total = (size_t)n_ids[i];
    const size_t keep = total >= cut_front + cut_back ? total - cut_front - cut_back : 0;
    results[i].len = keep;
    results[i].token_ids = static_cast<int*>(malloc(sizeof(int) * (keep ? keep : 1)));
    if (results[i].token_ids) memcpy(results[i].token_ids, ids.data() + i * (size_t)stride + cut_front, sizeof(int) * keep);
    else results[i].len = 0;
  }
}

}  // namespace

extern "C" {

TokenizerHandle tokenizers_new_from_path(const char* path) {
  if (!path) return nullptr;
  return make(path);
}

TokenizerHandle tokenizers_new_from_str(const char* data, size_t len) {
  if (!data || !len) return nullptr;
  char name[] = "/tmp/xllm_tokenizer_XXXXXX";
  const int fd = mkstemp(name);
  if (fd < 0) return nullptr;
  FILE* f = fdopen(fd, "wb");
  const bool ok = f && fwrite(data, 1, len, f) == len;
  if (f) fclose(f);
  LegacyTokenizer* L = ok ? make(name) : nullptr;
  remove(name);
  return L;
}

void tokenizers_encode(TokenizerHandle handle, const char* data, size_t len, int add_special_token,
                       TokenizerEncodeResult* result) {
  if (!result) return;
  encode_many(static_cast<LegacyTokenizer*>(handle), &data, &len, 1, add_special_token != 0, result);
}

void tokenizers_encode_batch(TokenizerHandle handle, const char* const* data, const size_t* len, size_t num_seqs,
                             int add_special_token, TokenizerEncodeResult* results) {
  if (!results) return;
  encode_many(static_cast<LegacyTokenizer*>(handle), data, len, num_seqs, add_special_token != 0, results);
}

void tokenizers_free_encode_results(TokenizerEncodeResult* results, size_t num_seqs) {
  if (!results) return;
  for (size_t i = 0; i < num_seqs; ++i) {
    free(results[i].token_ids);
    results[i].token_ids = nullptr;
    results[i].len = 0;
  }
}

void tokenizers_decode(TokenizerHandle handle, const uint32_t* data, size_t len, int skip_special_tokens,
                       const char** decode_data, size_t* decode_len) {
  LegacyTokenizer* L = static_cast<LegacyTokenizer*>(handle);
  if (!L || !decode_data || !decode_len) return;
  L->scratch = decode_ids(*L->h->sp_tables, data, len, skip_special_tokens != 0);
  *decode_data = L->scratch.data();
  *decode_len = L->scratch.size();
}

void tokenizers_id_to_token(TokenizerHandle handle, uint32_t id, const char** data, size_t* len) {
  LegacyTokenizer* L = static_cast<LegacyTokenizer*>(handle);
  if (!L || !data || !len) return;
  const xllm::SpTables& t = *L->h->sp_tables;
  L->scratch = id < t.piece_str.size() ? t.piece_str[id] : std::string();
  *data = L->scratch.data();
  *len = L->scratch.size();
}

void tokenizers_token_to_id(TokenizerHandle handle, const char* token, size_t len, int32_t* id) {
  LegacyTokenizer* L = static_cast<LegacyTokenizer*>(handle);
  if (!id) return;
  *id = -1;
  if (!L || !token) return;
  auto it = L->piece_to_id.find(std::string(token, len));
  if (it != L->piece_to_id.end()) *id = it->second;
}

void tokenizers_free(TokenizerHandle handle) {
  LegacyTokenizer* L = static_cast<LegacyTokenizer*>(handle);
  if (!L) return;
  xllm_ingest_destroy(L->h);
  delete L;
}

void tokenizers_get_vocab_size(TokenizerHandle handle, size_t* size) {
  LegacyTokenizer* L = static_cast<LegacyTokenizer*>(handle);
  if (!size) return;
  *size = 0;
  if (L) {
    const xllm::SpTables& t = *L->h->sp_tables;
    *size = t.vocab_size_override >= 0 ? (size_t)t.vocab_size_override : (size_t)t.n_pieces;
  }
}

}  // extern "C"
