// sp_encode.cuh — device-resident SentencePiece-BPE tables + the batched encode kernel launcher.
//
// Device replacement for Tokenizer::encode on the SentencePiece backend
// (xllm_service/tokenizer/tokenizer.h:32-33, sentencepiece_tokenizer.cpp:115-168; called per
// request at xllm_service/scheduler/scheduler.cpp:129).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sp_model.h"

namespace xllm {

// Pointers into device memory, passed to the kernel by value (__grid_constant__).
struct SpDev {
  const uint32_t* trie;
  const uint8_t* blob;
  const uint32_t* ascii_sym;
  const CpEntry* cp_table;
  const PairEntry* pair_table;
  const int32_t* emit;
  const uint32_t* virt_cp;
  const int32_t* byte_id;
  uint32_t trie_units;
  uint32_t cp_mask;
  uint32_t pair_mask;
  uint32_t pair_shift;  // 32 - log2(pair slots): the slot is the hash's top bits
  uint32_t n_pieces;
  uint32_t space_sym;
  int32_t unk_id;
  uint32_t max_unit_out;
  uint32_t simple_ascii[4];
  uint32_t spacelike_ascii[4];  // bytes the charsmap turns into exactly one space (SpTables::spacelike_ascii)
  uint8_t byte_fallback, add_dummy_prefix, remove_extra_ws, split_mode;
  uint8_t small_vocab;  // ranks and piece ids fit 16 bits: packed merge scratch
  uint8_t byte_mode;    // tiktoken tables: every byte is a symbol, text is copied verbatim
  uint8_t printable_simple;  // every byte 0x20..0x7E is "simple" (simple_ascii): word-at-a-time fast-path test
  uint8_t express;           // express_step allowed (XLLM_SP_EXPRESS=0 turns it off)
  // global scratch pool for pre-tokens too long for shared memory (sp_long_word.cuh)
  // HF byte-level BPE (split_mode 3, hf_model.cc): Unicode classes for the GPT-2 regex, the added (special)
  // tokens matched verbatim in the text, and the template ids wrapped around every sequence
  const uint16_t* uni1;
  const uint8_t* uni2;
  const uint8_t* added_blob;
  const uint16_t* added_off;  // [n_added + 1]
  const int32_t* added_id;
  uint32_t n_added, added_max_len;
  uint32_t n_added_plain;     // != 0: added[0, n_added_plain) are matched first, the rest only between them (MODE 3)
  uint32_t added_first[8];    // bit b set <=> some added token starts with byte b
  int32_t prefix_ids[4], suffix_ids[4];
  uint8_t n_prefix, n_suffix;
  uint8_t ignore_merges;  // a pre-token that is a vocabulary entry is emitted as that id (vtab / vblob)
  const uint4* vtab;
  const uint8_t* vblob;
  uint32_t vtab_mask;
  // Unigram SentencePiece: Viterbi over vtab (NORMAL pieces) with piece_score; see unigram_word (sp_encode.cu)
  uint8_t unigram;
  const float* piece_score;
  float unk_score;
  uint32_t max_piece_len;
  const uint4* utrie;   // byte trie of the pieces: {parent, byte, child, piece id or -1}, parent 0xFFFFFFFF = empty
  uint32_t utrie_mask;
  uint8_t nfc_check;   // normalizer NFC: a request passes only if NFC provably leaves it unchanged: every char is
                       // NFC-inert, or (nfc_verdict set) the verify kernel found it in NFC
  // normalizer NFC, exact verification (hf_nfc.cu; uploaded for nfc_check models, scripts/gen_unicode_nfc.py):
  // {ccc, NFC_Quick_Check} per code point (two-stage), full canonical decompositions, primary composites
  const uint16_t* nfc1;
  const uint16_t* nfc2;
  const uint32_t* nfc_decomp_cp;         // ascending
  const uint32_t* nfc_decomp;            // 4 per entry, 0-padded
  const unsigned long long* nfc_comp_key;  // first << 21 | second, ascending
  const uint32_t* nfc_comp;
  uint32_t n_nfc_decomp, n_nfc_comp;
  uint8_t hf_pattern;  // 1: ByteLevel's own GPT-2 regex, 2: Split(cl100k-family regex) + ByteLevel(use_regex = false)
  uint8_t hf_digits;   // pattern 2: \p{N}{1,hf_digits}
  // per-launch options (set by sp_encode_launch from SpLaunchOpts; null = off)
  const uint8_t* nfc_verdict;    // [n_req] verdicts of hf_nfc_verify_kernel (0 NFC, 1 not NFC, 2 malformed UTF-8):
                                 // the inert-char proof is skipped and a refused request is not tokenised
  const int64_t* out_start;      // request r's ids go to ids + out_start[r] (at most out_cap[r]) instead of r * ids_stride
  const int32_t* out_cap;
  unsigned long long* warp_ns;   // [grid]: nanoseconds each warp of the throughput kernel spent from start to exit
  uint8_t* warm_arena;           // [grid] slices of kWarmSliceBytes: scratch of the warm-up pre-passes (sp_encode.cu drain_pass 1b)
  const int32_t* work_list;      // buffer-path kernel after the express kernel: the requests handed over, their count,
  const unsigned int* work_count;  // and where each one resumes (ExpResume records, sp_encode.cu)
  const void* resume;
  uint8_t* long_pool;
  int* long_locks;
  uint32_t long_cap;   // symbols per slot
  int32_t long_slots;
};

// Per-request status written by the kernel.
constexpr int32_t kEncOk = 0;
constexpr int32_t kEncTruncated = 1;     // more ids than ids_stride: n_ids holds the full count, the row its prefix
constexpr int32_t kEncBadUtf8 = -1;      // HF backend: the text is not valid UTF-8 (the reference's Rust shim panics)
constexpr int32_t kEncNeedsNfc = -5;     // HF backend with normalizer NFC: the text is not provably in NFC (XLLM_ERR_UNSUPPORTED)
                                         // or, verifying, not in NFC / holds a Maybe chunk over kNfcChunkCap code points
constexpr int32_t kEncWordTooLong = -6;  // a single pre-token exceeds the on-chip word capacity (XLLM_ERR_CAPACITY)

class SpDeviceModel {
 public:
  ~SpDeviceModel();
  int upload(const SpTables& t);  // XLLM_OK or error (set_last_error)
  const SpDev& dev() const { return dev_; }

 private:
  SpDev dev_{};
  void* allocs_[32] = {nullptr};
  int n_allocs_ = 0;
};

// Word memo: a write-once hash table word bytes -> token ids that lives for ONE launch (the launcher clears
// it first), so a word that occurs again in the same batch skips symbol building, pair probes and the merge.
// 32 bytes per slot; slots = power of two; table == nullptr disables it.
struct SpMemo {
  void* table = nullptr;
  uint32_t slots = 0;
  // false: the launch reuses what earlier launches left in the table (same tokenizer model; entries are immutable, so a
  // stale table is only ever less complete) — the caller's policy decides when to clear (xllm_set_memo_policy)
  bool clear = true;
  // true: run the warm-up pre-passes (natural text: memo misses merged in full rounds, long words resolved ahead of
  // the in-order rounds); arena is their scratch, at least SpEncodePlan::arena_bytes
  bool warm = false;
  void* arena = nullptr;
  size_t arena_bytes = 0;
};
uint32_t sp_memo_default_slots();  // XLLM_SP_MEMO_SLOTS (0 = off), default 2^18 = 8 MiB

// What one sp_encode_launch over n_req requests runs, and the device memory it needs.
struct SpEncodePlan {
  bool memo = false;       // the throughput kernel uses the word memo
  bool warm = false;       // ... with the warm-up pre-passes (BPE models, memo on)
  bool express = false;    // the express kernel runs first (memo on, not warm, sp_express_model)
  bool long_pass = false;  // the long-word kernel runs last, over the deferred requests (BPE models)
  int kernels = 0;         // kernels enqueued
  int express_blocks = 0;  // blocks of the express kernel ...
  int express_warps = 0;   // ... of this many warps (at most its block shape, sp_encode.cu ExpShape)
  int grid = 0;            // warps (= blocks) of the buffer-path throughput kernel: as many as its shared memory lets
                           // the SMs hold, at most n_req
  int grid_long = 0;       // warps of the long-word kernel
  int warp_ns = 0;         // SpLaunchOpts::warp_ns entries: the larger of the two throughput grids, in warps
  bool nfc_verify = false; // hf_nfc_verify_kernel runs first (asked for, and the model has normalizer NFC)
  int nfc_blocks = 0;      // its blocks of kNfcWarps warps
  size_t scratch_bytes = 0;  // sp_encode_launch's scratch (+ one verdict byte per request when nfc_verify)
  size_t arena_bytes = 0;    // warm: SpMemo::arena for the full grid (any n_req), else 0
};
cudaError_t sp_encode_plan(const SpDev& dev, int n_req, bool memo, bool warm, SpEncodePlan* plan,
                           bool nfc_verify = false);

// text: all prompts back to back; offsets[n_req + 1] (bytes).  Request r's ids go to
// ids + r * ids_stride (at most ids_stride of them), n_ids[r] = full count, status[r] = kEnc*.
// counters: 8 uint32 in device memory; scratch: SpEncodePlan::scratch_bytes of device memory (work lists of the
// follow-up kernels + resume records).  Launches the kernels sp_encode_plan lists (no-op grids when there is nothing
// to do); a warm launch whose arena is smaller than the plan's fails with cudaErrorInvalidValue.
struct SpLaunchOpts {
  // ragged output rows (text pieces of segmented requests, pipeline.cu): ids + out_start[r], capacity out_cap[r]
  const int64_t* out_start = nullptr;
  const int32_t* out_cap = nullptr;
  // diagnostics: per-warp busy time of the throughput kernels' persistent grids (SpEncodePlan::warp_ns entries);
  // used by bench.py to report the length tail of variable-length batches
  unsigned long long* warp_ns = nullptr;
  // normalizer NFC: verify each request exactly (hf_nfc.cu) instead of proving every char NFC-inert
  // (xllm_set_nfc_policy); no effect on other models.  Plan with the same flag.
  bool nfc_verify = false;
};
cudaError_t sp_encode_launch(const SpDev& dev, const uint8_t* text, const int64_t* offsets, int n_req, int32_t* ids,
                             int64_t ids_stride, int32_t* n_ids, int32_t* status, unsigned int* counters,
                             void* scratch, cudaStream_t stream, SpMemo memo = SpMemo(),
                             SpLaunchOpts opts = SpLaunchOpts());

// Exact NFC verification (hf_nfc.cu): one warp per request, blocks of kNfcWarps warps; verdict[r] = 0 in NFC, 1 not in
// NFC or a chunk holding an NFC_QC = Maybe char is longer than kNfcChunkCap code points, 2 malformed UTF-8.
// task_counter: one zeroed uint32 in device memory.
constexpr int kNfcChunkCap = 32;
constexpr int kNfcWarps = 4;
cudaError_t hf_nfc_verify_launch(const SpDev& dev, const uint8_t* text, const int64_t* offsets, int n_req,
                                 uint8_t* verdict, unsigned int* task_counter, int blocks, cudaStream_t stream);

}  // namespace xllm
