// hf_model.cc — HF `tokenizer.json` (byte-level BPE) -> the device tables of the encode kernels.
//
// Host-side replacement of what FastTokenizer delegates to the Rust `tokenizers` crate
// (xllm_service/tokenizer/fast_tokenizer.cpp:8-30 -> tokenizers_new_from_path / tokenizers_encode,
// xllm_service/tokenizer/tokenizers/src/lib.rs:56-99), chosen by the factory whenever
// <dir>/tokenizer.json exists (tokenizer_factory.cpp:14-19).
//
// Supported configuration (everything else fails the load with XLLM_ERR_UNSUPPORTED — never a silent
// approximation): model BPE without dropout / unk / prefix / suffix / byte_fallback / ignore_merges;
// normalizer null; pre_tokenizer one of the layouts in hf_load_model's kLayouts (GPT-2 ByteLevel, cl100k-family
// Split, DeepSeek-V3's three Splits);
// post_processor null, ByteLevel, or a TemplateProcessing whose `single` template only wraps the sequence in
// special tokens; added tokens without lstrip/rstrip/single_word, matched verbatim: the normalized:false ones first,
// the normalized:true ones between those (under normalizer NFC only NFC-inert normalized contents are taken, so
// NFC(content) = content).
// Tables: byte_mode (every byte is a symbol: the byte-level alphabet is a bijection byte <-> char), the pair
// table comes straight from `merges` (priority = merge rank), split_mode 3 = the regex pre-tokenizer.
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "common.cuh"
#include "sp_model.h"

namespace xllm {

uint32_t sp_pair_slot(uint32_t a, uint32_t b, uint32_t n_slots);

namespace {

#include "unicode_classes.inc"

// ------------------------------------------------------------------ a small JSON reader
struct JVal {
  enum Type { kNull, kBool, kNum, kStr, kArr, kObj } type = kNull;
  bool b = false;
  double num = 0;
  std::string str;
  std::vector<JVal> arr;
  std::vector<std::pair<std::string, JVal>> obj;
  const JVal* get(const char* key) const {
    for (const auto& kv : obj)
      if (kv.first == key) return &kv.second;
    return nullptr;
  }
  bool is_null() const { return type == kNull; }
};

class JParser {
 public:
  JParser(const char* p, const char* e) : p_(p), e_(e) {}
  bool parse(JVal* out) { return value(out, 0) && (ws(), true); }

 private:
  void ws() { while (p_ < e_ && (*p_ == ' ' || *p_ == '\n' || *p_ == '\t' || *p_ == '\r')) ++p_; }
  static void put_utf8(uint32_t cp, std::string* s) {
    if (cp < 0x80) s->push_back((char)cp);
    else if (cp < 0x800) { s->push_back((char)(0xC0 | (cp >> 6))); s->push_back((char)(0x80 | (cp & 0x3F))); }
    else if (cp < 0x10000) { s->push_back((char)(0xE0 | (cp >> 12))); s->push_back((char)(0x80 | ((cp >> 6) & 0x3F))); s->push_back((char)(0x80 | (cp & 0x3F))); }
    else { s->push_back((char)(0xF0 | (cp >> 18))); s->push_back((char)(0x80 | ((cp >> 12) & 0x3F))); s->push_back((char)(0x80 | ((cp >> 6) & 0x3F))); s->push_back((char)(0x80 | (cp & 0x3F))); }
  }
  bool hex4(uint32_t* v) {
    if (e_ - p_ < 4) return false;
    *v = 0;
    for (int i = 0; i < 4; ++i) {
      const char c = *p_++;
      *v <<= 4;
      if (c >= '0' && c <= '9') *v |= c - '0';
      else if (c >= 'a' && c <= 'f') *v |= c - 'a' + 10;
      else if (c >= 'A' && c <= 'F') *v |= c - 'A' + 10;
      else return false;
    }
    return true;
  }
  bool string(std::string* s) {
    if (p_ >= e_ || *p_ != '"') return false;
    ++p_;
    while (p_ < e_ && *p_ != '"') {
      if (*p_ == '\\') {
        if (++p_ >= e_) return false;
        const char c = *p_++;
        switch (c) {
          case 'n': s->push_back('\n'); break;
          case 't': s->push_back('\t'); break;
          case 'r': s->push_back('\r'); break;
          case 'b': s->push_back('\b'); break;
          case 'f': s->push_back('\f'); break;
          case 'u': {
            uint32_t cp;
            if (!hex4(&cp)) return false;
            if (cp >= 0xD800 && cp < 0xDC00 && e_ - p_ >= 6 && p_[0] == '\\' && p_[1] == 'u') {
              p_ += 2;
              uint32_t lo;
              if (!hex4(&lo)) return false;
              cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
            }
            put_utf8(cp, s);
            break;
          }
          default: s->push_back(c);  // \" \\ \/
        }
      } else {
        s->push_back(*p_++);
      }
    }
    if (p_ >= e_) return false;
    ++p_;
    return true;
  }
  bool value(JVal* v, int depth) {
    if (depth > 64) return false;
    ws();
    if (p_ >= e_) return false;
    const char c = *p_;
    if (c == '{') {
      v->type = JVal::kObj;
      ++p_;
      ws();
      if (p_ < e_ && *p_ == '}') { ++p_; return true; }
      for (;;) {
        ws();
        std::string k;
        if (!string(&k)) return false;
        ws();
        if (p_ >= e_ || *p_++ != ':') return false;
        v->obj.emplace_back(std::move(k), JVal());
        if (!value(&v->obj.back().second, depth + 1)) return false;
        ws();
        if (p_ < e_ && *p_ == ',') { ++p_; continue; }
        if (p_ < e_ && *p_ == '}') { ++p_; return true; }
        return false;
      }
    }
    if (c == '[') {
      v->type = JVal::kArr;
      ++p_;
      ws();
      if (p_ < e_ && *p_ == ']') { ++p_; return true; }
      for (;;) {
        v->arr.emplace_back();
        if (!value(&v->arr.back(), depth + 1)) return false;
        ws();
        if (p_ < e_ && *p_ == ',') { ++p_; continue; }
        if (p_ < e_ && *p_ == ']') { ++p_; return true; }
        return false;
      }
    }
    if (c == '"') { v->type = JVal::kStr; return string(&v->str); }
    if (e_ - p_ >= 4 && !strncmp(p_, "true", 4)) { v->type = JVal::kBool; v->b = true; p_ += 4; return true; }
    if (e_ - p_ >= 5 && !strncmp(p_, "false", 5)) { v->type = JVal::kBool; v->b = false; p_ += 5; return true; }
    if (e_ - p_ >= 4 && !strncmp(p_, "null", 4)) { v->type = JVal::kNull; p_ += 4; return true; }
    char* end = nullptr;
    v->num = strtod(p_, &end);
    if (end == p_ || end > e_) return false;
    v->type = JVal::kNum;
    p_ = end;
    return true;
  }
  const char* p_;
  const char* e_;
};

// GPT-2 bytes_to_unicode: byte -> code point of its printable stand-in
void byte_level_alphabet(uint32_t cp_of_byte[256]) {
  bool direct[256] = {false};
  for (int b = '!'; b <= '~'; ++b) direct[b] = true;
  for (int b = 0xA1; b <= 0xAC; ++b) direct[b] = true;
  for (int b = 0xAE; b <= 0xFF; ++b) direct[b] = true;
  int n = 0;
  for (int b = 0; b < 256; ++b) cp_of_byte[b] = direct[b] ? (uint32_t)b : (uint32_t)(256 + n++);
}
std::string utf8_of(uint32_t cp) {
  std::string s;
  if (cp < 0x80) s.push_back((char)cp);
  else if (cp < 0x800) { s.push_back((char)(0xC0 | (cp >> 6))); s.push_back((char)(0x80 | (cp & 0x3F))); }
  else { s.push_back((char)(0xE0 | (cp >> 12))); s.push_back((char)(0x80 | ((cp >> 6) & 0x3F))); s.push_back((char)(0x80 | (cp & 0x3F))); }
  return s;
}

// the bytes a token spelled in the byte-level alphabet stands for; false when a char is outside the alphabet
bool byte_level_bytes(const std::string& tok, const std::unordered_map<uint32_t, uint8_t>& byte_of_cp, std::string* raw) {
  const uint8_t* p = (const uint8_t*)tok.data();
  const size_t n = tok.size();
  size_t i = 0;
  raw->clear();
  while (i < n) {
    uint32_t cp;
    if (p[i] < 0x80) { cp = p[i]; i += 1; }
    else if ((p[i] & 0xE0) == 0xC0 && i + 1 < n) { cp = ((p[i] & 0x1F) << 6) | (p[i + 1] & 0x3F); i += 2; }
    else if ((p[i] & 0xF0) == 0xE0 && i + 2 < n) { cp = ((p[i] & 0x0F) << 12) | ((p[i + 1] & 0x3F) << 6) | (p[i + 2] & 0x3F); i += 3; }
    else return false;
    auto it = byte_of_cp.find(cp);
    if (it == byte_of_cp.end()) return false;
    raw->push_back((char)it->second);
  }
  return true;
}

int fail(SpTables* t, int code, const std::string& msg) {
  t->error = msg;
  return code;
}

bool flag_false_or_absent(const JVal* o, const char* key) {
  const JVal* v = o ? o->get(key) : nullptr;
  return !v || v->is_null() || (v->type == JVal::kBool && !v->b);
}

// pre_tokenizer ByteLevel{add_prefix_space: false} with use_regex (default true) as wanted
bool byte_level_ok(const JVal& bl, bool want_regex) {
  const JVal* bt = bl.get("type");
  const JVal* rx = bl.get("use_regex");
  const bool use_regex = !(rx && rx->type == JVal::kBool && !rx->b);
  return bt && bt->type == JVal::kStr && bt->str == "ByteLevel" && flag_false_or_absent(&bl, "add_prefix_space") &&
         use_regex == want_regex;
}

// pre_tokenizer Split{pattern: {Regex}, behavior: Isolated, invert: false} -> its regex; null for any other entry
const std::string* split_regex(const JVal& sp) {
  const JVal* st = sp.get("type");
  const JVal* pat = sp.get("pattern");
  const JVal* rx = pat ? pat->get("Regex") : nullptr;
  const JVal* beh = sp.get("behavior");
  if (!st || st->type != JVal::kStr || st->str != "Split" || !rx || rx->type != JVal::kStr || !beh ||
      beh->type != JVal::kStr || beh->str != "Isolated" || !flag_false_or_absent(&sp, "invert"))
    return nullptr;
  return &rx->str;
}

}  // namespace

// The top-level string member `key` of a JSON file, as the reference's JsonReader::value<std::string>(key) reads it
// (tokenizer_args.cpp:49-51): a key of that name nested in another object (auto_map, processor ...) does not count.
bool json_file_top_level_string(const std::string& path, const char* key, std::string* out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  std::string js;
  char buf[4096];
  size_t got;
  while ((got = fread(buf, 1, sizeof(buf), f)) > 0) js.append(buf, got);
  fclose(f);
  JVal root;
  JParser parser(js.data(), js.data() + js.size());
  if (!parser.parse(&root) || root.type != JVal::kObj) return false;
  const JVal* v = root.get(key);
  if (!v || v->type != JVal::kStr) return false;
  *out = v->str;
  return true;
}

bool tokenizer_dir_has_hf_json(const std::string& dir) {
  struct stat st;
  return stat((dir + "/tokenizer.json").c_str(), &st) == 0 && S_ISREG(st.st_mode);
}

int hf_load_model(const std::string& path_in, SpTables* t) {
  std::string path = path_in;
  struct stat st;
  if (stat(path.c_str(), &st) == 0 && S_ISDIR(st.st_mode)) path += "/tokenizer.json";
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return fail(t, XLLM_ERR_IO, "cannot open " + path);
  std::string js;
  char buf[1 << 16];
  size_t got;
  while ((got = fread(buf, 1, sizeof(buf), f)) > 0) js.append(buf, got);
  fclose(f);
  JVal root;
  if (!JParser(js.data(), js.data() + js.size()).parse(&root) || root.type != JVal::kObj)
    return fail(t, XLLM_ERR_FORMAT, path + ": not a JSON object");
  const JVal* model = root.get("model");
  if (!model || model->type != JVal::kObj || !model->get("vocab") || !model->get("merges"))
    return fail(t, XLLM_ERR_FORMAT, path + ": no model.vocab / model.merges");
  const JVal* mtype = model->get("type");
  if (mtype && mtype->type == JVal::kStr && mtype->str != "BPE")
    return fail(t, XLLM_ERR_UNSUPPORTED, "tokenizer.json model type " + mtype->str + ": only BPE is supported on device");
  for (const char* k : {"dropout", "unk_token", "continuing_subword_prefix", "end_of_word_suffix"}) {
    const JVal* v = model->get(k);
    if (v && !v->is_null() && !(v->type == JVal::kStr && v->str.empty()))
      return fail(t, XLLM_ERR_UNSUPPORTED, std::string("tokenizer.json model.") + k + " is not supported on device");
  }
  t->ignore_merges = !flag_false_or_absent(model, "ignore_merges");
  for (const char* k : {"fuse_unk", "byte_fallback"})
    if (!flag_false_or_absent(model, k))
      return fail(t, XLLM_ERR_UNSUPPORTED, std::string("tokenizer.json model.") + k + " = true is not supported on device");
  const JVal* norm = root.get("normalizer");
  if (norm && !norm->is_null()) {
    // NFC (Qwen2 family): the device proves per request that NFC is the identity (every char NFC-inert) and
    // fails the request otherwise — it never normalises
    const JVal* ty = norm->get("type");
    const JVal* members = norm->get("normalizers");
    const bool empty_sequence = ty && ty->type == JVal::kStr && ty->str == "Sequence" && members &&
                                members->type == JVal::kArr && members->arr.empty();   // DeepSeek-V3 ships this no-op
    if (!empty_sequence) {
      if (!ty || ty->type != JVal::kStr || ty->str != "NFC")
        return fail(t, XLLM_ERR_UNSUPPORTED, "tokenizer.json normalizer: only null, an empty Sequence or NFC is supported on device");
      t->nfc_check = true;
    }
  }
  for (const char* k : {"truncation", "padding"}) {
    const JVal* v = root.get(k);
    if (v && !v->is_null()) return fail(t, XLLM_ERR_UNSUPPORTED, std::string("tokenizer.json ") + k + " is not supported on device");
  }
  const JVal* pre = root.get("pre_tokenizer");
  {
    static const char* kUnsupported =
        "tokenizer.json pre_tokenizer: supported on device are ByteLevel{add_prefix_space:false, use_regex:true}, "
        "Sequence[Split{cl100k-family regex, Isolated}, ByteLevel{add_prefix_space:false, use_regex:false}] and the "
        "DeepSeek-V3 Sequence[Split{\\p{N}{1,3}}, Split{CJK/kana runs}, Split{main regex}, ByteLevel{use_regex:false}]";
    // DeepSeek-V3 / R1 (scheduler/xllm_chat_parse_bridge.cpp:49-78 names the family): three Isolated splits
    static const char* kDs1 = "\\p{N}{1,3}";
    static const char* kDs2 = "[\xe4\xb8\x80-\xe9\xbe\xa5\xe3\x81\x80-\xe3\x82\x9f\xe3\x82\xa0-\xe3\x83\xbf]+";
    static const char* kDs3 =
        "[!\"#$%&'()*+,\\-./:;<=>?@\\[\\\\\\]^_`{|}~][A-Za-z]+|[^\r\n\\p{L}\\p{P}\\p{S}]?[\\p{L}\\p{M}]+| ?[\\p{P}\\p{S}]+[\r\n]*|"
        "\\s*[\r\n]+|\\s+(?!\\S)|\\s+";
    static const char* kP3 =
        "(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\\r\\n\\p{L}\\p{N}]?\\p{L}+|\\p{N}{1,3}| ?[^\\s\\p{L}\\p{N}]+[\\r\\n]*|\\s*[\\r\\n]+|\\s+(?!\\S)|\\s+";
    static const char* kP1 =
        "(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\\r\\n\\p{L}\\p{N}]?\\p{L}+|\\p{N}| ?[^\\s\\p{L}\\p{N}]+[\\r\\n]*|\\s*[\\r\\n]+|\\s+(?!\\S)|\\s+";
    // the accepted layouts: the Split regexes in order, then ByteLevel, with its own regex only when there is no Split
    struct Layout {
      size_t n_splits;
      const char* splits[3];
      int pattern, digits;
    };
    static const Layout kLayouts[] = {
        {0, {}, 1, 3},                   // GPT-2: a bare ByteLevel
        {1, {kP3}, 2, 3},                // cl100k family, Llama-3
        {1, {kP1}, 2, 1},                // cl100k family, Qwen2
        {3, {kDs1, kDs2, kDs3}, 3, 3},   // DeepSeek-V3 / R1
    };
    const JVal* ty = pre ? pre->get("type") : nullptr;
    const JVal* seq = pre ? pre->get("pretokenizers") : nullptr;
    const bool is_seq = ty && ty->type == JVal::kStr && ty->str == "Sequence" && seq && seq->type == JVal::kArr &&
                        seq->arr.size() >= 2;
    if (!is_seq && !(ty && ty->type == JVal::kStr && ty->str == "ByteLevel")) return fail(t, XLLM_ERR_UNSUPPORTED, kUnsupported);
    const size_t n_splits = is_seq ? seq->arr.size() - 1 : 0;
    if (!byte_level_ok(is_seq ? seq->arr.back() : *pre, !is_seq)) return fail(t, XLLM_ERR_UNSUPPORTED, kUnsupported);
    std::vector<const std::string*> regex(n_splits);
    for (size_t k = 0; k < n_splits; ++k)
      if (!(regex[k] = split_regex(seq->arr[k]))) return fail(t, XLLM_ERR_UNSUPPORTED, kUnsupported);
    const Layout* layout = nullptr;
    size_t matched = 0;   // the most leading Split entries that a layout of this length accepts
    for (const Layout& l : kLayouts) {
      if (l.n_splits != n_splits) continue;
      size_t k = 0;
      while (k < n_splits && *regex[k] == l.splits[k]) ++k;
      if (k == n_splits) layout = &l;
      matched = std::max(matched, k);
    }
    if (!layout) return fail(t, XLLM_ERR_UNSUPPORTED, std::string(kUnsupported) + "; got regex " + *regex[matched]);
    t->hf_pattern = layout->pattern;
    t->hf_digits = layout->digits;
  }

  // ---- vocabulary
  const JVal* vocab = model->get("vocab");
  if (vocab->type != JVal::kObj || vocab->obj.empty()) return fail(t, XLLM_ERR_FORMAT, "model.vocab is not an object");
  std::unordered_map<std::string, int32_t> id_of;
  int32_t max_id = -1;
  for (const auto& kv : vocab->obj) {
    if (kv.second.type != JVal::kNum) return fail(t, XLLM_ERR_FORMAT, "model.vocab value is not a number");
    const int32_t id = (int32_t)kv.second.num;
    if (id < 0 || id >= 0x3FFFFFFF) return fail(t, XLLM_ERR_FORMAT, "model.vocab id out of range");
    id_of.emplace(kv.first, id);
    max_id = id > max_id ? id : max_id;
  }
  // ---- added tokens, with the ids `tokenizers` gives them when it loads the file (AddedVocabulary::add_tokens, in
  // list order) whatever ids the file lists: a content that is a model.vocab entry or an earlier added token keeps
  // that id, any other gets len(model.vocab), or one past the largest added id once that is at least len(model.vocab)
  struct Added {
    std::string content;
    int32_t id;
    bool special, normalized;
  };
  std::vector<Added> added_list;
  std::unordered_map<std::string, int32_t> added_id_of;
  const JVal* added = root.get("added_tokens");
  if (added && added->type == JVal::kArr) {
    int32_t top = -1;
    for (const JVal& a : added->arr) {
      const JVal* content = a.get("content");
      const JVal* id = a.get("id");
      if (!content || content->type != JVal::kStr || content->str.empty() || !id || id->type != JVal::kNum)
        return fail(t, XLLM_ERR_FORMAT, "bad added_tokens entry");
      if (!flag_false_or_absent(&a, "single_word") || !flag_false_or_absent(&a, "lstrip") ||
          !flag_false_or_absent(&a, "rstrip"))
        return fail(t, XLLM_ERR_UNSUPPORTED, "added token '" + content->str + "': single_word/lstrip/rstrip are not supported on device");
      if (content->str.size() > 64) return fail(t, XLLM_ERR_UNSUPPORTED, "added token longer than 64 bytes");
      const bool special = !flag_false_or_absent(&a, "special");
      const JVal* nz = a.get("normalized");
      const bool normalized = nz && nz->type == JVal::kBool ? nz->b : !special;   // the library's default
      if (added_id_of.count(content->str)) {
        // an identical repeat is ignored, as the library does; one with other flags would make them depend on the
        // library's bookkeeping (the special set keeps the first, the id's entry the last)
        for (const auto& b : added_list)
          if (b.content == content->str && (b.special != special || b.normalized != normalized))
            return fail(t, XLLM_ERR_UNSUPPORTED, "added token '" + content->str + "' is listed twice with different flags");
        continue;
      }
      // `normalized` tokens are matched in the second pass on the text itself: with normalizer NFC the device only
      // encodes text NFC leaves unchanged, and the library matches NFC(content) there, so a content is taken only when
      // every char of it is NFC-inert (then NFC(content) = content)
      if (normalized && t->nfc_check) {
        const uint8_t* u = (const uint8_t*)content->str.data();
        for (size_t i = 0; i < content->str.size();) {
          uint32_t cp = u[i];
          int l = 1;
          if (cp >= 0xF0) { cp &= 0x07; l = 4; } else if (cp >= 0xE0) { cp &= 0x0F; l = 3; } else if (cp >= 0xC0) { cp &= 0x1F; l = 2; }
          for (int k = 1; k < l && i + k < content->str.size(); ++k) cp = (cp << 6) | (u[i + k] & 0x3F);
          i += l;
          if (cp >= 0x80 && cp < 0x110000 && (kUniStage2[(size_t)kUniStage1[cp >> 8] * 256 + (cp & 255)] & 4))
            return fail(t, XLLM_ERR_UNSUPPORTED, "normalized added token '" + content->str + "' is not NFC-inert under normalizer NFC");
        }
      }
      auto in_vocab = id_of.find(content->str);
      const int32_t aid = in_vocab != id_of.end() ? in_vocab->second
                          : (top < (int32_t)id_of.size() ? (int32_t)id_of.size() : top + 1);
      top = std::max(top, aid);
      added_id_of.emplace(content->str, aid);
      added_list.push_back(Added{content->str, aid, special, normalized});
      max_id = aid > max_id ? aid : max_id;
    }
    {   // the device keeps them in one blob addressed by 16-bit offsets (DeepSeek-V3: ~820 tokens, ~25 KB)
      size_t blob = 0;
      for (const auto& a : added_list) blob += a.content.size();
      if (added_list.size() > 2048 || blob > 65535)
        return fail(t, XLLM_ERR_UNSUPPORTED, "added tokens: more than 2048 of them or more than 65535 bytes in total");
    }
    // the non-normalized tokens first: the device matches added_tokens[0, n_added_plain) in its first pass
    for (int pass = 0; pass < 2; ++pass)
      for (const auto& a : added_list)
        if (a.normalized == (pass == 1)) t->added_tokens.emplace_back(a.content, a.id);
    for (const auto& a : added_list) t->n_added_plain += !a.normalized;
  }
  const uint32_t V = (uint32_t)max_id + 1;
  t->byte_mode = true;
  t->split_mode = 3;
  t->add_dummy_prefix = false;
  t->remove_extra_whitespaces = false;
  t->byte_fallback = false;
  t->unk_id = -1;
  t->max_unit_out = 4;
  t->n_pieces = V;
  t->n_syms = V;
  t->emit.assign(V, -2);
  for (const auto& kv : id_of) t->emit[(size_t)kv.second] = kv.second;
  t->virt_cp.assign(1, 0);
  t->byte_id.assign(256, -1);
  t->cp_table.assign(16, CpEntry{kEmptyKey, 0});
  t->space_sym = kEmptyKey;
  // byte -> symbol of its byte-level char
  uint32_t cp_of_byte[256];
  byte_level_alphabet(cp_of_byte);
  std::unordered_map<uint32_t, uint8_t> byte_of_cp;
  t->ascii_sym.assign(256, 0);
  for (int b = 0; b < 256; ++b) {
    byte_of_cp.emplace(cp_of_byte[b], (uint8_t)b);
    auto it = id_of.find(utf8_of(cp_of_byte[b]));
    if (it == id_of.end()) return fail(t, XLLM_ERR_UNSUPPORTED, "the byte-level alphabet is not fully in model.vocab");
    t->ascii_sym[b] = (uint32_t)it->second;
  }
  // decode table: token string (byte-level chars) -> raw bytes
  t->piece_str.assign(V, std::string());
  t->piece_raw.assign(V, std::string());
  std::vector<bool> raw_ok(V, false);
  t->piece_type.assign(V, 1);
  for (const auto& kv : id_of) {
    std::string raw;
    const bool ok = byte_level_bytes(kv.first, byte_of_cp, &raw);
    t->piece_str[(size_t)kv.second] = kv.first;
    t->piece_raw[(size_t)kv.second] = ok ? raw : kv.first;
    raw_ok[(size_t)kv.second] = ok;
  }
  if (t->ignore_merges) {
    // raw bytes of every model.vocab entry -> id, probed once per pre-token on device (hf_vocab_lookup)
    std::vector<std::pair<std::string, int32_t>> ent;
    for (const auto& kv : id_of) {
      // an entry spelled with chars outside the byte alphabet can never equal a byte-level pre-token
      if (raw_ok[(size_t)kv.second]) ent.emplace_back(t->piece_raw[(size_t)kv.second], kv.second);
    }
    const int rc = build_bytes_table(ent, t);
    if (rc != XLLM_OK) return rc;
  }
  size_t n_extra = 0;
  for (const auto& a : added_list) {
    n_extra += id_of.find(a.content) == id_of.end();
    t->piece_str[(size_t)a.id] = a.content;
    // the ByteLevel decoder maps an added token like any other: to bytes when all its chars are in the byte
    // alphabet, verbatim otherwise
    std::string raw;
    if (!byte_level_bytes(a.content, byte_of_cp, &raw)) raw = a.content;
    t->piece_raw[(size_t)a.id] = raw;
    t->piece_type[(size_t)a.id] = a.special ? 3 : 1;  // 3: skipped by decode(skip_special_tokens)
    if ((size_t)a.id < t->emit.size()) t->emit[(size_t)a.id] = a.id;
  }
  t->vocab_size_override = (int32_t)(id_of.size() + n_extra);  // Tokenizer::get_vocab_size(with_added_tokens = true), lib.rs
  // ---- merges -> pair table (priority = index)
  const JVal* merges = model->get("merges");
  if (merges->type != JVal::kArr) return fail(t, XLLM_ERR_FORMAT, "model.merges is not an array");
  std::vector<PairEntry> pairs;
  pairs.reserve(merges->arr.size());
  for (size_t i = 0; i < merges->arr.size(); ++i) {
    const JVal& m = merges->arr[i];
    std::string a, b;
    if (m.type == JVal::kArr && m.arr.size() == 2 && m.arr[0].type == JVal::kStr && m.arr[1].type == JVal::kStr) {
      a = m.arr[0].str;
      b = m.arr[1].str;
    } else if (m.type == JVal::kStr) {
      const size_t sp = m.str.find(' ');
      if (sp == std::string::npos) return fail(t, XLLM_ERR_FORMAT, "bad merges entry");
      a = m.str.substr(0, sp);
      b = m.str.substr(sp + 1);
    } else {
      return fail(t, XLLM_ERR_FORMAT, "bad merges entry");
    }
    auto ia = id_of.find(a), ib = id_of.find(b), iab = id_of.find(a + b);
    if (ia == id_of.end() || ib == id_of.end() || iab == id_of.end())
      return fail(t, XLLM_ERR_FORMAT, "merge '" + a + " " + b + "' refers to a token outside model.vocab");
    pairs.push_back(PairEntry{(uint32_t)ia->second, (uint32_t)ib->second, (uint32_t)i, (uint32_t)iab->second});
  }
  uint32_t n = 16;
  while (n < pairs.size() * 4 + 16) n <<= 1;
  t->pair_table.assign(n, PairEntry{kEmptyKey, kEmptyKey, kNoPrio, 0});
  for (const auto& e : pairs) {
    uint32_t h = sp_pair_slot(e.a, e.b, n);
    bool dup = false;
    while (t->pair_table[h].a != kEmptyKey) {
      if (t->pair_table[h].a == e.a && t->pair_table[h].b == e.b) { dup = true; break; }  // first (lowest) rank wins
      h = (h + 1) & (n - 1);
    }
    if (!dup) t->pair_table[h] = e;
  }
  // ---- post-processor: ids wrapped around the sequence when add_special_tokens = 1 (fast_tokenizer.cpp:24).
  // ByteLevel only trims offsets; a Sequence (Llama-3: [ByteLevel, TemplateProcessing]) applies its members in order.
  {
    std::vector<const JVal*> procs;
    const JVal* post = root.get("post_processor");
    if (post && !post->is_null()) {
      const JVal* ty = post->get("type");
      if (!ty || ty->type != JVal::kStr) return fail(t, XLLM_ERR_FORMAT, "post_processor without a type");
      if (ty->str == "Sequence") {
        const JVal* list = post->get("processors");
        if (!list || list->type != JVal::kArr) return fail(t, XLLM_ERR_FORMAT, "post_processor Sequence without processors");
        for (const JVal& x : list->arr) procs.push_back(&x);
      } else {
        procs.push_back(post);
      }
    }
    bool have_template = false;
    for (const JVal* pr : procs) {
      const JVal* ty = pr->get("type");
      if (!ty || ty->type != JVal::kStr) return fail(t, XLLM_ERR_FORMAT, "post_processor without a type");
      if (ty->str == "ByteLevel") continue;
      if (ty->str != "TemplateProcessing" || have_template)
        return fail(t, XLLM_ERR_UNSUPPORTED, "post_processor " + ty->str + " is not supported on device");
      have_template = true;
      const JVal* single = pr->get("single");
      const JVal* specials = pr->get("special_tokens");
      if (!single || single->type != JVal::kArr) return fail(t, XLLM_ERR_FORMAT, "TemplateProcessing without `single`");
      bool seen_seq = false;
      for (const JVal& it : single->arr) {
        if (const JVal* sq = it.get("Sequence")) {
          const JVal* id = sq->get("id");
          if (seen_seq || !id || id->type != JVal::kStr || id->str != "A")
            return fail(t, XLLM_ERR_UNSUPPORTED, "TemplateProcessing.single must contain sequence A exactly once");
          seen_seq = true;
        } else if (const JVal* st = it.get("SpecialToken")) {
          const JVal* id = st->get("id");
          const JVal* def = (specials && id && id->type == JVal::kStr) ? specials->get(id->str.c_str()) : nullptr;
          const JVal* ids = def ? def->get("ids") : nullptr;
          if (!ids || ids->type != JVal::kArr) return fail(t, XLLM_ERR_FORMAT, "TemplateProcessing special token without ids");
          for (const JVal& x : ids->arr) (seen_seq ? t->suffix_ids : t->prefix_ids).push_back((int32_t)x.num);
        } else {
          return fail(t, XLLM_ERR_UNSUPPORTED, "unsupported TemplateProcessing item");
        }
      }
      if (!seen_seq) return fail(t, XLLM_ERR_UNSUPPORTED, "TemplateProcessing.single without sequence A");
      if (t->prefix_ids.size() > 4 || t->suffix_ids.size() > 4)
        return fail(t, XLLM_ERR_UNSUPPORTED, "more than 4 template tokens on one side");
    }
  }
  // ---- Unicode classes for the regex (\p{L}, \p{N}, \s)
  t->uni_stage1.assign(kUniStage1, kUniStage1 + sizeof(kUniStage1) / sizeof(kUniStage1[0]));
  t->uni_stage2.assign(kUniStage2, kUniStage2 + sizeof(kUniStage2));
  return XLLM_OK;
}

}  // namespace xllm
