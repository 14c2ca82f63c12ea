// sp_model.h — host-side loader that turns a SentencePiece `.model` (BPE) into the flat
// device tables the encode kernel walks.
//
// Replaces what SentencePieceTokenizer's constructor does through libsentencepiece
// (xllm_service/tokenizer/sentencepiece_tokenizer.cpp:43-54: sp_processor_.Load(<dir>/tokenizer.model)).
#pragma once
#include <stdint.h>

#include <string>
#include <utility>
#include <vector>

namespace xllm {

constexpr uint32_t kSymUnknownFlag = 0x80000000u;  // sym = flag | codepoint : a char no piece contains
constexpr uint32_t kEmptyKey = 0xFFFFFFFFu;
constexpr uint32_t kNoPrio = 0xFFFFFFFFu;

struct PairEntry {  // 16 bytes: one LDG.128 per probe
  uint32_t a, b;    // left / right symbol; a == kEmptyKey marks an empty slot
  uint32_t prio;    // merge priority: rank of the merged piece's score, 0 = highest score (merges first)
  uint32_t merged;  // symbol of the concatenation
};
struct CpEntry {
  uint32_t cp;   // Unicode code point, kEmptyKey = empty
  uint32_t sym;  // its symbol
};

// Everything the kernel needs, as host vectors (uploaded verbatim).
struct SpTables {
  // normalizer (NormalizerSpec.precompiled_charsmap = Darts double array + NUL-separated replacements)
  std::vector<uint32_t> trie;
  std::vector<uint8_t> blob;
  uint32_t max_unit_out = 3;  // max bytes one normalisation unit can append to the normalized stream
  // bit b set <=> ASCII byte b is "simple": the charsmap has no key that is exactly b and every longer key
  // starting with b continues with a byte >= 0x80, so b followed by an ASCII byte normalises to itself
  uint32_t simple_ascii[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
  // ASCII bytes the charsmap rewrites to exactly one space (tab, LF, CR ... under nmt_nfkc) and that start no longer
  // key continuing with an ASCII byte: the fast path treats them as a source space (bit b of word b >> 5)
  uint32_t spacelike_ascii[4] = {0, 0, 0, 0};
  bool add_dummy_prefix = true;
  bool remove_extra_whitespaces = true;
  // symbols: [0, n_pieces) = piece ids; [n_pieces, n_syms) = single chars that occur inside
  // pieces (or are reserved single-char pieces) without being NORMAL pieces themselves
  uint32_t n_pieces = 0, n_syms = 0;
  std::vector<uint32_t> ascii_sym;  // [128]
  std::vector<CpEntry> cp_table;    // open addressing, power-of-two size
  std::vector<PairEntry> pair_table;
  std::vector<int32_t> emit;        // [n_syms]: token id, or -1 = unknown (byte fallback / unk)
  std::vector<uint32_t> virt_cp;    // [n_syms - n_pieces] code point of each virtual symbol
  std::vector<int32_t> byte_id;     // [256] ids of <0x00>..<0xFF> (all -1 without byte_fallback)
  int32_t unk_id = 0;
  bool byte_fallback = false;
  uint32_t space_sym = 0;  // symbol of U+2581
  // 0: no exact pre-split exists (whole text is one word); 1: split before every U+2581;
  // 2: split before a U+2581 unless the previous char is U+2581 too
  int split_mode = 1;
  // tiktoken tables (tiktoken_model.cc): every BYTE is a symbol (ascii_sym has 256 entries), no normaliser,
  // no whitespace rules; emit == -2 marks a symbol that produces no id
  bool byte_mode = false;
  int32_t vocab_size_override = -1;
  // HF byte-level BPE (hf_model.cc): split_mode 3 = the GPT-2 regex pre-tokenizer over the raw bytes;
  // added tokens are matched verbatim in the text, the first n_added_plain (normalized: false) in a first pass, the
  // rest (normalized: true) in a second pass between those; template ids wrap every sequence
  std::vector<std::pair<std::string, int32_t>> added_tokens;
  uint32_t n_added_plain = 0;
  std::vector<int32_t> prefix_ids, suffix_ids;
  int hf_pattern = 1;   // 1: ByteLevel's own GPT-2 regex, 2: Split(cl100k-family regex) + ByteLevel(use_regex = false)
  int hf_digits = 3;    // pattern 2: \p{N}{1,hf_digits}
  bool ignore_merges = false;  // a pre-token that is a vocabulary entry is emitted as that id (models/bpe/model.rs)
  std::vector<uint32_t> vocab_table;  // ignore_merges: 4 x u32 per slot {hash lo, hash hi, id, blob offset << 10 | length}
  std::vector<uint8_t> vocab_blob;
  // Unigram SentencePiece (sp_model.cc): Viterbi over the vocabulary table above (NORMAL pieces) with these scores
  bool unigram = false;
  std::vector<float> piece_score;  // [n_pieces]
  float unk_score = 0.f;           // min NORMAL score - 10 (unigram_model.cc kUnkPenalty)
  uint32_t max_piece_len = 0;      // longest NORMAL piece in bytes
  // byte trie of the NORMAL pieces as a hash table (parent node, byte) -> (child node, piece id or -1):
  // 4 x u32 per slot {parent, byte, child, piece}, parent 0xFFFFFFFF = empty; node 0 is the root
  std::vector<uint32_t> uni_trie;
  bool nfc_check = false;      // normalizer NFC: requests are accepted only when NFC leaves them unchanged
  std::vector<uint16_t> uni_stage1;  // [0x1100]  code point >> 8 -> block
  std::vector<uint8_t> uni_stage2;   // [blocks * 256] class: 0 other, 1 \p{L}, 2 \p{N}, 3 \s
  // vocabulary strings for decode / id_to_token / token_to_id
  std::vector<std::string> piece_str;
  std::vector<std::string> piece_raw;  // HF byte-level: the bytes each token decodes to (piece_str keeps the vocab spelling)
  std::vector<uint8_t> piece_type;
  std::string error;
};

// Fills vocab_table / vocab_blob: raw bytes -> id, probed on device by hf_vocab_lookup (hf_pretok.cuh): FNV-1a 64
// of the bytes, slot from the mixed hash, 16-byte entries {hash lo, hash hi, id, blob offset << 10 | length}.
// Returns XLLM_OK or XLLM_ERR_UNSUPPORTED (an entry longer than 512 bytes / more than 4 MiB of bytes).
int build_bytes_table(const std::vector<std::pair<std::string, int32_t>>& entries, SpTables* t);
// Loads <path> (file, or directory containing tokenizer.model).  Returns XLLM_OK or an error code
// (message in out->error).
int sp_load_model(const std::string& path, SpTables* out);
// tiktoken vocabulary (`base64(token) rank` lines) -> the same tables, byte_mode (tiktoken_model.cc)
int tiktoken_load_model(const std::string& path, SpTables* out);
// <dir>/tokenizer_config.json has "tokenizer_class": "TikTokenTokenizer" (tokenizer_factory.cpp:20-25)
bool tokenizer_dir_is_tiktoken(const std::string& dir);
bool json_file_top_level_string(const std::string& path, const char* key, std::string* out);   // hf_model.cc
// HF `tokenizer.json` byte-level BPE -> the same tables, byte_mode + split_mode 3 (hf_model.cc)
int hf_load_model(const std::string& path, SpTables* out);
// <dir>/tokenizer.json exists (tokenizer_factory.cpp:14-19: it wins over everything else)
bool tokenizer_dir_has_hf_json(const std::string& dir);
// the factory's choice for a tokenizer directory / file
int load_tokenizer_tables(const std::string& path, SpTables* out);

}  // namespace xllm
