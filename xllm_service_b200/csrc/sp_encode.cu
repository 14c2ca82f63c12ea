// sp_encode.cu — the batched tokenizer kernels on sm_90a: one warp per request.
//
// Bit-exact target: what Tokenizer::encode returns on each of the reference's backends —
//   SentencePiece (sentencepiece_tokenizer.cpp:115-168 -> sp_processor_.Encode):
//     normalizer.cc     Normalize(): longest-prefix rewrite through the precompiled charsmap trie,
//                       invalid UTF-8 -> U+FFFD, whitespace collapse, ' ' -> U+2581, dummy prefix
//     bpe_model.cc      Encode(): merge the adjacent pair with the best score, leftmost on ties,
//                       until no adjacent pair concatenates to a NORMAL piece
//     unigram_model.cc  EncodeOptimized(): Viterbi over the piece lattice (unigram_word below)
//     sentencepiece_processor.cc  byte fallback / consecutive-unknown merging
//   tiktoken in the service's regex-less mode (tiktoken_tokenizer.cpp:115-294): byte symbols, merges by rank
//   HF `tokenizer.json` byte-level BPE (fast_tokenizer.cpp:20-30): hf_pretok.cuh in front of the same merges
//
// Two throughput kernels.  sp_express_kernel (SentencePiece BPE models with split_mode 1 + remove_extra_whitespaces,
// memo on) tokenises 512-byte windows of plain ASCII text straight from the loaded bytes — no normalized-text buffer,
// no word list: lane k takes the window's words k and k + 32, probes the word memo for both at once and stores the ids
// from the memo payloads (express_run below).  What its rules do not cover is handed to
// sp_encode_kernel, the general kernel described next, which is also the only kernel of every other backend.
//
// Why the BPE merge is exact AND parallel: no NORMAL piece of the loaded model holds U+2581 anywhere but
// at its first char (checked by the host loader: SpTables::split_mode), so no merge can ever
// span the boundary in front of a U+2581.  The priority-ordered global merge therefore factors
// into independent per-"word" merges.  The warp streams the request through shared memory:
//   1. normalise into a 2 KB normalized-text buffer: 128 source bytes per step on the ASCII fast path
//      (one word-at-a-time test per lane), 32 per step on the general path (every lane walks the trie
//      from its own byte; a ballot resolves which positions start a unit);
//   2. when the buffer fills, split it at U+2581 and hand one word per lane: the lane first probes the
//      per-launch word memo (word bytes -> ids); on a miss it builds its symbols (chars -> symbol ids),
//      looks up every adjacent pair in the (left,right) -> (priority, merged) hash table in L2, runs the
//      serial best-pair merge over a column of shared memory (alive bitmask in a register) and inserts
//      the result; words of 17..512 chars are merged by the whole warp cooperatively, longer ones in a
//      global scratch slot by a second launch;
//   3. ids are written straight to the request's output row in order.
// Algorithmic HBM traffic: text bytes read once + 4 B per id written.
#include "sp_encode.cuh"

#include <stdlib.h>
#include <string.h>

#include <type_traits>
#include <vector>

#include "common.cuh"
#include "sp_long_word.cuh"

namespace xllm {

namespace {

constexpr int kNBuf = 2048;        // normalized-text staging buffer per warp (bytes)
constexpr int kFastWin = 128;      // source bytes per fast-path step (4 per lane)
constexpr int kExpWin = 512;       // source bytes per express step (16 per lane)
constexpr int kPrefetchFirst = 2;  // fast path: prefetch windows pos + 2 .. pos + 2 + kPrefetchWindows - 1 into L2
constexpr int kPrefetchWindows = 2;
constexpr int kLongEnterAt = 1024;   // a kept tail (one incomplete word) longer than this switches to long mode
constexpr int kLongFlushAt = 1024;   // long mode: move nbuf into the scratch slot once it holds this much
constexpr int kMaxSym = 16;        // lane-per-word path: chars per word (alive set = 16 bits of a register)
constexpr int kCoopMaxSym = 512;   // warp-cooperative path: chars per word (= 32 * kMaxSym scratch entries)
constexpr int kMaxWords = 704;     // >= kNBuf / 3 + 2 word starts
constexpr uint32_t kFull = 0xffffffffu;
// per-warp slice of the launch's warm-up scratch (global, L2-resident): ids of pre-resolved long words, addressed by
// the word's byte offset in nbuf (a word never yields more ids than it has bytes), + their id counts per word index
constexpr size_t kWarmSliceBytes = (size_t)kNBuf * 4 + (size_t)kMaxWords * 2;
constexpr uint16_t kNotPre = 0xFFFFu;
constexpr uint32_t kResolvedFlag = 0x40000000u;  // S[] entry holds a token id, not a symbol (bit 31 clear)

// (priority, merged symbol) of the pair starting at a position.  SMALL (ranks and piece ids < 65535):
// packed into one u32 so a warp's merge scratch is 8 KB instead of 12 KB (more resident warps per SM).
template <bool SMALL>
struct PMOps;
template <>
struct PMOps<false> {
  using T = uint2;
  static constexpr uint32_t kNone = kNoPrio;
  static __device__ __forceinline__ T pack(uint2 v) { return v; }
  static __device__ __forceinline__ T none() { return make_uint2(kNoPrio, 0); }
  static __device__ __forceinline__ uint32_t prio(T v) { return v.x; }
  static __device__ __forceinline__ uint32_t merged(T v) { return v.y; }
  static __device__ __forceinline__ uint32_t prio_at(const T* p) { return p->x; }
};
template <>
struct PMOps<true> {
  using T = uint32_t;
  static constexpr uint32_t kNone = 0xFFFFu;
  static __device__ __forceinline__ T pack(uint2 v) { return v.x == kNoPrio ? 0xFFFF0000u : ((v.x << 16) | v.y); }
  static __device__ __forceinline__ T none() { return 0xFFFF0000u; }
  static __device__ __forceinline__ uint32_t prio(T v) { return v >> 16; }
  static __device__ __forceinline__ uint32_t merged(T v) { return v & 0xFFFFu; }
  // the priority half alone, straight from shared memory (one LDS.U16, no shift)
  static __device__ __forceinline__ uint32_t prio_at(const T* p) {
    return reinterpret_cast<const uint16_t*>(p)[1];
  }
};

// ROWS = chars per word on the lane-per-word path (the lane's column height).  16 for the warm-up and Unigram kernels;
// the buffer-path BPE kernels take 32 (kHfRows, first measured on the HF byte-level kernels): natural text through a byte-level BPE has 10 % of its pre-tokens between 17 and 32
// bytes, and a 32-row column keeps them on the lane path (32 words merged at once) instead of the one-word-at-a-time
// cooperative path — at the price of 8 KB more shared memory per warp (17 / 13 resident warps instead of 27 / 18).
constexpr int kHfRows = 32;
template <bool SMALL, int ROWS = kMaxSym>
struct WarpSmemT {
  static constexpr int kRows = ROWS;
  static constexpr int kSyms = ROWS * 32 > kCoopMaxSym ? ROWS * 32 : kCoopMaxSym;
  uint32_t S[kSyms];                   // symbols: lane columns S[j * 32 + lane] (lane path) or flat (cooperative)
  typename PMOps<SMALL>::T PM[kSyms];  // pair state at position j
  uint8_t nbuf[kNBuf];                       // normalized text (always starts at a word start)
  uint16_t wstart[kMaxWords];
  uint16_t pend[32];                         // warm-up kernels: words that missed the memo, waiting for a full round
};
// Unigram kernels: plus the pieces found from each of 32 start positions (unigram_word)
constexpr int kUniMaxMatch = 32;
template <bool SMALL>
struct WarpSmemUniT : WarpSmemT<SMALL> {
  uint32_t mlist[32 * kUniMaxMatch];  // [start lane][k]: piece id (24 bits, 0xFFFFFF = unknown char) | length << 24
};

__device__ __forceinline__ uint32_t hash_pair(uint32_t a, uint32_t b) {
  return (a * 0x9E3779B1u + b) * 0x85EBCA6Bu;  // multiplicative; the slot is its top bits (sp_model.cc)
}
__device__ __forceinline__ uint32_t hash_cp(uint32_t cp) {
  uint32_t h = cp * 0x9E3779B1u;
  h ^= h >> 16;
  return h;
}

// (left, right) -> (priority, merged); priority kNoPrio when A||B is not a piece.
// Split in two so callers can put several first probes in flight before consuming any of them.
struct PairProbe {
  uint32_t h;
  uint4 e;
};
__device__ __forceinline__ PairProbe pair_probe_begin(const SpDev& T, uint32_t a, uint32_t b) {
  PairProbe p;
  p.h = hash_pair(a, b) >> T.pair_shift;
  p.e = ((a | b) & kSymUnknownFlag) ? make_uint4(kEmptyKey, 0, 0, 0)
                                    : __ldg(reinterpret_cast<const uint4*>(T.pair_table) + p.h);
  return p;
}
__device__ __forceinline__ uint2 pair_probe_finish(const SpDev& T, uint32_t a, uint32_t b, PairProbe p) {
  for (;;) {
    if (p.e.x == a && p.e.y == b) return make_uint2(p.e.z, p.e.w);
    if (p.e.x == kEmptyKey) return make_uint2(kNoPrio, 0);
    p.h = (p.h + 1) & T.pair_mask;
    p.e = __ldg(reinterpret_cast<const uint4*>(T.pair_table) + p.h);
  }
}
__device__ __forceinline__ uint2 pair_lookup(const SpDev& T, uint32_t a, uint32_t b) {
  return pair_probe_finish(T, a, b, pair_probe_begin(T, a, b));
}

__device__ __forceinline__ uint32_t cp_lookup(const SpDev& T, uint32_t cp) {
  if (cp == 0x2581u) return T.space_sym;
  uint32_t h = hash_cp(cp) & T.cp_mask;
  for (;;) {
    const uint2 e = __ldg(reinterpret_cast<const uint2*>(T.cp_table) + h);
    if (e.x == cp) return e.y;
    if (e.x == kEmptyKey) return kSymUnknownFlag | cp;
    h = (h + 1) & T.cp_mask;
  }
}

// util.cc DecodeUTF8 + IsValidDecodeUTF8 on p[0..avail): returns bytes to consume, sets valid.
__device__ __forceinline__ uint32_t utf8_unit(const uint8_t* p, uint32_t avail, uint8_t b0, bool* valid) {
  *valid = true;
  if (b0 < 0x80) return 1;
  auto trail = [](uint8_t x) { return (x & 0xC0) == 0x80; };
  if (avail >= 2 && (b0 & 0xE0) == 0xC0) {
    const uint8_t b1 = p[1];
    const uint32_t cp = ((b0 & 0x1Fu) << 6) | (b1 & 0x3Fu);
    if (trail(b1) && cp >= 0x80) return 2;
  } else if (avail >= 3 && (b0 & 0xF0) == 0xE0) {
    const uint8_t b1 = p[1], b2 = p[2];
    const uint32_t cp = ((b0 & 0x0Fu) << 12) | ((b1 & 0x3Fu) << 6) | (b2 & 0x3Fu);
    if (trail(b1) && trail(b2) && cp >= 0x800 && !(cp >= 0xD800 && cp < 0xE000)) return 3;
  } else if (avail >= 4 && (b0 & 0xF8) == 0xF0) {
    const uint8_t b1 = p[1], b2 = p[2], b3 = p[3];
    const uint32_t cp = ((b0 & 0x07u) << 18) | ((b1 & 0x3Fu) << 12) | ((b2 & 0x3Fu) << 6) | (b3 & 0x3Fu);
    if (trail(b1) && trail(b2) && trail(b3) && cp >= 0x10000 && cp <= 0x10FFFF) return 4;
  }
  *valid = false;  // malformed: consume one byte, emit U+FFFD
  return 1;
}

// Char at p (well-formed by construction: normalized text) -> symbol; *adv = its byte length.
__device__ __forceinline__ uint32_t char_sym(const SpDev& T, const uint8_t* p, uint32_t* adv) {
  const uint32_t b0 = p[0];
  if (b0 < 0x80 || T.byte_mode) {  // byte_mode (tiktoken tables): every byte is a symbol, 256-entry table
    *adv = 1;
    return __ldg(T.ascii_sym + b0);
  }
  uint32_t cp, l;
  if (b0 < 0xE0) { l = 2; cp = ((b0 & 0x1F) << 6) | (p[1] & 0x3F); }
  else if (b0 < 0xF0) { l = 3; cp = ((b0 & 0x0F) << 12) | ((p[1] & 0x3Fu) << 6) | (p[2] & 0x3F); }
  else { l = 4; cp = ((b0 & 0x07) << 18) | ((p[1] & 0x3Fu) << 12) | ((p[2] & 0x3Fu) << 6) | (p[3] & 0x3F); }
  *adv = l;
  return cp_lookup(T, cp);
}

// Token ids of one final symbol.  Returns the count (1..4), ids in out[]; *unk = symbol is unknown.
__device__ __forceinline__ int sym_ids(const SpDev& T, uint32_t sym, int32_t out[4], bool* unk) {
  uint32_t cp;
  *unk = false;
  if (!(sym & kSymUnknownFlag)) {
    const int32_t e = __ldg(T.emit + sym);
    if (e >= 0) { out[0] = e; return 1; }
    if (e == -2) return 0;  // a part without a rank is skipped (tiktoken_tokenizer.cpp:228-229)
    cp = __ldg(T.virt_cp + (sym - T.n_pieces));
  } else {
    cp = sym & 0x1FFFFFu;
  }
  *unk = true;
  if (!T.byte_fallback) { out[0] = T.unk_id; return 1; }
  uint8_t b[4];
  int n;
  if (cp < 0x80) { b[0] = (uint8_t)cp; n = 1; }
  else if (cp < 0x800) { b[0] = 0xC0 | (cp >> 6); b[1] = 0x80 | (cp & 0x3F); n = 2; }
  else if (cp < 0x10000) { b[0] = 0xE0 | (cp >> 12); b[1] = 0x80 | ((cp >> 6) & 0x3F); b[2] = 0x80 | (cp & 0x3F); n = 3; }
  else { b[0] = 0xF0 | (cp >> 18); b[1] = 0x80 | ((cp >> 12) & 0x3F); b[2] = 0x80 | ((cp >> 6) & 0x3F); b[3] = 0x80 | (cp & 0x3F); n = 4; }
  for (int i = 0; i < n; ++i) out[i] = __ldg(T.byte_id + b[i]);
  return n;
}

__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(kFull, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

#include "hf_pretok.cuh"

// ---------------------------------------------------------------------------- word memo
// Slot = two 16-byte halves, each read / written with ONE morally-strong 128-bit access:
//   half 0  key: byte 0 = (starts with U+2581) << 7 | n, bytes 1..n = the word's bytes (without that U+2581), 0-padded
//   half 1  ids: x = 1 << 31 | count << 28 | id0, y z w = id1..id3      (count 1..4, ids < 2^28), or, when every
//           id fits 16 bits (SMALL tables): eight u16 = {0x8000 | count, id0 .. id6}  (count 1..7)
// Write-once per launch: a slot is claimed by a 128-bit CAS of its key over zero, then its ids are stored; a reader
// that finds its key but zero ids treats the word as a miss.  No slot is ever rewritten while a launch runs, so
// a key match binds the ids to that key exactly (no tags, no probabilistic checks).
struct U128 {
  unsigned long long lo, hi;
};
__device__ __forceinline__ U128 ld_b128(const void* p) {
  U128 v;
  asm volatile("{.reg .b128 t; ld.relaxed.gpu.global.b128 t, [%2]; mov.b128 {%0,%1}, t; }"
               : "=l"(v.lo), "=l"(v.hi) : "l"(p) : "memory");
  return v;
}
// The same load without the .relaxed.gpu qualifier, so that the SM's L1 may serve it: the express kernel's memo probes
// (exp_probe_finish).  An aligned 16-byte load returns one whole 16-byte value that was stored there, possibly an
// older one than L2 holds, and every value a slot half ever holds gives the exact result: zero or another word's key
// is a miss (the lane merges the word, and its insert finds the key, when it is already there); the word's key with
// zero ids is a miss; the word's key with its ids is a hit.  A launch writes each half at most once, from zero.
__device__ __forceinline__ U128 ld_b128_cached(const void* p) {
  U128 v;
  asm volatile("{.reg .b128 t; ld.global.b128 t, [%2]; mov.b128 {%0,%1}, t; }"
               : "=l"(v.lo), "=l"(v.hi) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_b128(void* p, U128 v) {
  asm volatile("{.reg .b128 t; mov.b128 t, {%1,%2}; st.relaxed.gpu.global.b128 [%0], t; }"
               :: "l"(p), "l"(v.lo), "l"(v.hi) : "memory");
}
__device__ __forceinline__ U128 cas_b128(void* p, U128 cmp, U128 val) {
  U128 o;
  asm volatile("{.reg .b128 c, n, o; mov.b128 c, {%3,%4}; mov.b128 n, {%5,%6}; "
               "atom.relaxed.gpu.global.cas.b128 o, [%2], c, n; mov.b128 {%0,%1}, o; }"
               : "=l"(o.lo), "=l"(o.hi) : "l"(p), "l"(cmp.lo), "l"(cmp.hi), "l"(val.lo), "l"(val.hi) : "memory");
  return o;
}
template <bool SMALL>
struct MemoIds {
  static constexpr int kMax = SMALL ? 7 : 4;
  static __device__ __forceinline__ bool valid(U128 v) { return SMALL ? ((uint32_t)v.lo >> 15) & 1u : (uint32_t)v.lo >> 31; }
  static __device__ __forceinline__ int count(U128 v) { return SMALL ? (int)((uint32_t)v.lo & 7u) : (int)(((uint32_t)v.lo >> 28) & 7u); }
  static __device__ __forceinline__ uint32_t id(U128 v, int q) {  // q < count
    if (SMALL) {
      const int f = q + 1;  // u16 field index
      const unsigned long long w = f < 4 ? v.lo : v.hi;
      return (uint32_t)(w >> ((f & 3) * 16)) & 0xFFFFu;
    }
    return q == 0 ? ((uint32_t)v.lo & 0x0FFFFFFFu) : q == 1 ? (uint32_t)(v.lo >> 32) : q == 2 ? (uint32_t)v.hi : (uint32_t)(v.hi >> 32);
  }
  static __device__ __forceinline__ U128 pack(int k, const uint32_t* ids) {
    U128 v{0ull, 0ull};
    if (SMALL) {
      v.lo = 0x8000u | (uint32_t)k;
      for (int q = 0; q < k; ++q) {
        const int f = q + 1;
        if (f < 4) v.lo |= (unsigned long long)ids[q] << (f * 16);
        else v.hi |= (unsigned long long)ids[q] << ((f & 3) * 16);
      }
    } else {
      v.lo = (unsigned long long)(0x80000000u | ((uint32_t)k << 28) | ids[0]) | ((unsigned long long)ids[1] << 32);
      v.hi = (unsigned long long)ids[2] | ((unsigned long long)ids[3] << 32);
    }
    return v;
  }
};
constexpr int kMemoMaxKeyBytes = 15;

// Key of word nb[ws, we); false when the word cannot be memoised (empty after the prefix, or too long).
__device__ __forceinline__ bool memo_key(const uint8_t* nb, int ws, int we, bool byte_mode, U128* key) {
  uint32_t hdr = 0;
  if (!byte_mode && we - ws >= 3 && nb[ws] == 0xE2 && nb[ws + 1] == 0x96 && nb[ws + 2] == 0x81) { ws += 3; hdr = 0x80; }
  const int n = we - ws;
  if (n < 1 || n > kMemoMaxKeyBytes) return false;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(nb) + (ws >> 2);  // 16 bytes from ws (reads past nlen are masked)
  const uint32_t sh = (ws & 3) * 8;
  uint32_t b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    b[i] = __funnelshift_r(w[i], w[i + 1], sh);
    const int nb_i = n - 4 * i;
    if (nb_i < 4) b[i] = nb_i <= 0 ? 0u : (b[i] & ((1u << (8 * nb_i)) - 1u));
  }
  const unsigned long long lo = (unsigned long long)b[0] | ((unsigned long long)b[1] << 32);
  const unsigned long long hi = (unsigned long long)b[2] | ((unsigned long long)b[3] << 32);
  key->lo = (lo << 8) | (hdr | (uint32_t)n);
  key->hi = (hi << 8) | (lo >> 56);
  return true;
}
__device__ __forceinline__ uint32_t memo_slot(U128 k, uint32_t mask) {
  unsigned long long h = (k.lo ^ (k.hi * 0x9E3779B97F4A7C15ull)) * 0xD6E8FEB86659FD93ull;
  h ^= h >> 32;
  return (uint32_t)h & mask;
}

// State of one request while it streams through the warp.
struct ReqState {
  const uint8_t* src;
  uint32_t len;
  int32_t* out;
  int64_t cap;          // ids_stride
  int64_t n_out;        // ids produced so far (may exceed cap)
  int32_t nlen;         // bytes in nbuf
  int32_t trailing_bare;  // ids emitted by the current run of trailing bare-U+2581 words
  int32_t nw;           // word starts recorded so far in wstart[] (valid when !rescan)
  bool rescan;          // a general-path window ran since the last drain: word starts must be re-derived
  bool ascii;           // nbuf holds only ASCII and U+2581 (written by the fast path)
  bool prev_space;      // normalizer's is_prev_space
  bool prev_unk;        // last emitted symbol was unknown (byte_fallback off only)
  bool too_long;
  float uni_score;     // Unigram: best-path score at the start of the next word (running float, as upstream)
  int8_t bad_input;    // HF backend: 1 malformed UTF-8, 2 not provably NFC under a normalizer NFC
  bool deferred;       // needs the long-word kernel (this one was built without it)
  bool warm;           // warm-up kernels: the last drain had several memo misses
  bool had_long;       // warm-up kernels: the last drain had words beyond the lane columns
  // long-word mode: the current pre-token is being streamed into a global scratch slot
  bool long_mode;
  bool long_last_sp;   // the last char appended to the slot is U+2581
  int long_slot;
  uint32_t long_n;     // symbols appended so far
};

__device__ __forceinline__ void put_id(ReqState& rs, int64_t pos, int32_t id) {
  if (pos < rs.cap) rs.out[pos] = id;
}

// ---------------------------------------------------------------------------- normalisation
// Normalises source bytes [pos, pos + 32) (units that START in that window) and appends the result to nbuf.
// carry_skip: leading bytes of the window already consumed by the previous window's last unit.
template <typename SM>
__device__ __forceinline__ bool normalize_window(const SpDev& T, SM& sm, ReqState& rs, uint32_t pos,
                                                 uint32_t& carry_skip, int lane) {
  const uint32_t i = pos + lane;
  const bool inb = i < rs.len;
  const uint8_t* p = rs.src + i;
  const uint8_t b0 = inb ? __ldg(p) : 0;
  uint32_t consume = 1, kind = 0 /*0 identity, 1 blob, 2 U+FFFD*/, val = 0;
  if (inb) {
    uint32_t best_len = 0, best_val = 0;
    if (T.trie_units) {
      // Darts-clone commonPrefixSearch; libsentencepiece keeps the first 32 hits and takes the longest
      uint32_t node = 0;
      uint32_t unit = __ldg(T.trie);
      node ^= (unit >> 10) << ((unit & 0x200u) >> 6);
      uint32_t hits = 0;
      const uint32_t avail = rs.len - i;
      for (uint32_t k = 0; k < avail; ++k) {
        const uint32_t c = k == 0 ? b0 : __ldg(p + k);
        node ^= c;
        if (node >= T.trie_units) break;
        unit = __ldg(T.trie + node);
        if ((unit & 0x800000FFu) != c) break;
        node ^= (unit >> 10) << ((unit & 0x200u) >> 6);
        if (node >= T.trie_units) break;
        if ((unit >> 8) & 1u) {
          if (hits < 32) { best_len = k + 1; best_val = __ldg(T.trie + node) & 0x7FFFFFFFu; }
          ++hits;
        }
      }
    }
    if (best_len) {
      consume = best_len; kind = 1; val = best_val;
    } else {
      bool valid;
      consume = utf8_unit(p, rs.len - i, b0, &valid);
      kind = valid ? 0 : 2;
    }
  }
  // which positions start a unit
  uint32_t starts;
  const uint32_t n_in = rs.len - pos < 32 ? rs.len - pos : 32;
  const uint32_t in_mask = n_in == 32 ? kFull : ((1u << n_in) - 1);
  const uint32_t multi = __ballot_sync(kFull, inb && consume != 1);
  uint32_t q_end;
  if (multi == 0 && carry_skip == 0) {  // every unit is one byte: every position starts one
    starts = in_mask;
    q_end = n_in;
  } else {  // follow the chain of units (uniform across the warp)
    starts = 0;
    uint32_t q = carry_skip;
    while (q < n_in) {
      starts |= 1u << q;
      q += __shfl_sync(kFull, consume, q);
    }
    q_end = q;
  }
  const uint32_t new_carry = q_end >= 32 ? q_end - 32 : 0;  // only meaningful when another window follows
  const bool is_start = (starts >> lane) & 1u;

  // replacement attributes
  uint32_t rlen = 0, lead_sp = 0, n_sp = 0;
  bool ends_sp = false;
  if (is_start) {
    if (kind == 0) { rlen = consume; lead_sp = n_sp = (b0 == ' '); ends_sp = (b0 == ' '); }
    else if (kind == 2) { rlen = 3; }
    else {
      const uint8_t* r = T.blob + val;
      bool leading = true;
      uint8_t c, last = 0;
      while ((c = __ldg(r + rlen)) != 0) {
        if (c == ' ') { ++n_sp; if (leading) ++lead_sp; } else leading = false;
        last = c;
        ++rlen;
      }
      ends_sp = last == ' ';
    }
  }
  const bool nonempty = is_start && rlen > 0;
  const bool all_sp = nonempty && lead_sp == rlen;
  uint32_t strip = 0;
  bool new_prev_space = rs.prev_space;
  if (T.remove_extra_ws) {
    const uint32_t ne_mask = __ballot_sync(kFull, nonempty);
    const uint32_t set_mask = __ballot_sync(kFull, nonempty && (all_sp || ends_sp));
    const uint32_t below = ne_mask & ((1u << lane) - 1);
    const bool state_before = below ? ((set_mask >> (31 - __clz(below))) & 1u) : rs.prev_space;
    if (state_before) strip = lead_sp;
    if (ne_mask) new_prev_space = (set_mask >> (31 - __clz(ne_mask))) & 1u;
  }
  const int out_len = is_start ? (int)((rlen - strip) + 2 * (n_sp - strip)) : 0;
  const int incl = warp_incl_scan(out_len, lane);
  const int total = __shfl_sync(kFull, incl, 31);
  if (rs.nlen + total > kNBuf) return false;  // does not fit: the caller drains and retries this window
  carry_skip = new_carry;
  rs.prev_space = new_prev_space;
  if (out_len) {
    uint8_t* d = sm.nbuf + rs.nlen + (incl - out_len);
    const uint8_t* r = kind == 1 ? T.blob + val : p;
    for (uint32_t k = strip; k < rlen; ++k) {
      uint8_t c;
      if (kind == 2) c = k == 0 ? 0xEF : (k == 1 ? 0xBF : 0xBD);
      else c = __ldg(r + k);
      if (c == ' ') { d[0] = 0xE2; d[1] = 0x96; d[2] = 0x81; d += 3; }
      else { *d++ = c; }
    }
  }
  rs.nlen += total;
  rs.rescan = true;   // word starts of this window are not tracked incrementally
  rs.ascii = false;
  __syncwarp();
  return true;
}

// Fast path: 128 source bytes per step, 4 per lane, valid when every byte is a "simple" ASCII byte
// (SpTables::simple_ascii) and is followed by another ASCII byte: then every byte is its own unit and
// normalises to itself, so only the whitespace rules remain:  a space is dropped iff the byte before it
// is a space (is_prev_space), kept spaces become U+2581 and start a word.  Returns false (nothing done)
// when the window does not qualify.
template <typename SM>
__device__ __forceinline__ bool normalize_fast(const SpDev& T, SM& sm, ReqState& rs, uint32_t pos, int lane) {
  const uint32_t base = pos + 4u * lane;
  const uint32_t nvalid = base >= rs.len ? 0u : (rs.len - base < 4u ? rs.len - base : 4u);
  // The lane's 4 source bytes as one little-endian word.  Every lane loads the ALIGNED word that holds its first
  // byte (one coalesced 128-byte request per warp) and borrows the next lane's word for the unaligned remainder;
  // words are only read while they start before the end of the request (bytes outside it are masked).
  const uint8_t* win = rs.src + pos;
  const uint32_t off = (uint32_t)(reinterpret_cast<uintptr_t>(win) & 3u);
  const uint32_t* aw = reinterpret_cast<const uint32_t*>(win - off) + lane;
  const uint8_t* src_end = rs.src + rs.len;
  const uint32_t W = reinterpret_cast<const uint8_t*>(aw) < src_end ? __ldg(aw) : 0x61616161u;
  // the text is read once, front to back: pull the next windows' lines into L2 while this one is processed
  if (lane < kPrefetchWindows) {
    const uint8_t* pf = reinterpret_cast<const uint8_t*>(aw - lane) + (size_t)kFastWin * (kPrefetchFirst + lane);
    if (pf < src_end) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf));
  }
  uint32_t Wn = __shfl_down_sync(kFull, W, 1);
  if (lane == 31) Wn = reinterpret_cast<const uint8_t*>(aw + 1) < src_end ? __ldg(aw + 1) : 0x61616161u;
  uint32_t w = __funnelshift_r(W, Wn, off * 8u);
  if (nvalid < 4u) w = nvalid == 0u ? 0x61616161u : ((w & ((1u << (8u * nvalid)) - 1u)) | (0x61616161u << (8u * nvalid)));
  uint32_t nextb = __shfl_down_sync(kFull, w, 1) & 0xFFu;
  if (lane == 31) nextb = base + 4 < rs.len ? ((Wn >> (off * 8u)) & 0xFFu) : 0x61u;
  if (!T.byte_mode) {
    // all four bytes ASCII and "simple"; the byte after them ASCII too.  Printable ASCII is simple for every
    // ordinary charsmap (host flag): three SWAR tests; anything else takes the per-byte table.
    const bool ascii4 = (w & 0x80808080u) == 0u;
    bool ok = (nextb < 0x80 || nvalid < 4) && ascii4;
    bool fast_ok = false;
    if (T.printable_simple)
      fast_ok = ((((w | 0x80808080u) - 0x20202020u) & 0x80808080u) == 0x80808080u) &&  // every byte >= 0x20
                (((w + 0x01010101u) & 0x80808080u) == 0u);                               // every byte <= 0x7E
    if (!__all_sync(kFull, ok && fast_ok)) {
      // per byte: simple, or "space-like" (the charsmap rewrites it to exactly one space: tab / LF / CR under
      // nmt_nfkc) — a space-like byte is turned into 0x20 here and from then on IS a source space
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t bk = (w >> (8 * k)) & 0xFFu;
        const bool spl = (T.spacelike_ascii[(bk >> 5) & 3] >> (bk & 31)) & 1u;
        ok = ok && (spl || ((T.simple_ascii[(bk >> 5) & 3] >> (bk & 31)) & 1u));
        if (spl && k < (int)nvalid) w = (w & ~(0xFFu << (8 * k))) | (0x20u << (8 * k));
      }
      if (!__all_sync(kFull, ok)) return false;
    }
  }
  // spaces as a 4-bit mask (byte_mode: text is copied verbatim, a space is an ordinary byte)
  uint32_t sp4 = 0;
  if (!T.byte_mode) {
    const uint32_t x = w ^ 0x20202020u;
    const uint32_t z = ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);  // 0x80 in every zero byte of x
    sp4 = (((z >> 7) * 0x01020408u) >> 24) & 0xFu;
  }
  // is the byte before this lane's first byte a space?  (lanes before a valid lane are full)
  uint32_t prev_in = __shfl_up_sync(kFull, sp4 >> 3, 1) & 1u;
  if (lane == 0) {
    // remove_extra_whitespaces: the normalizer's is_prev_space; otherwise "the last emitted char is U+2581"
    const int nl = rs.nlen;
    prev_in = T.remove_extra_ws ? (uint32_t)rs.prev_space
                                : (uint32_t)(nl >= 3 && sm.nbuf[nl - 3] == 0xE2 && sm.nbuf[nl - 2] == 0x96 && sm.nbuf[nl - 1] == 0x81);
  }
  const bool buffer_empty = rs.nlen == 0;  // offset 0 is a word start by definition: do not record it twice
  const uint32_t valid4 = (1u << nvalid) - 1u;
  const uint32_t prevbits = ((sp4 << 1) | prev_in) & 0xFu;            // bit k: the byte before byte k is a space
  const uint32_t keep4 = valid4 & ~(T.remove_extra_ws ? (sp4 & prevbits) : 0u);   // a space after a space is dropped
  const uint32_t az4 = (buffer_empty && lane == 0) ? (keep4 & (0u - keep4)) : 0u;  // the byte that lands at offset 0
  const uint32_t start4 =
      keep4 & sp4 & ~az4 & (T.split_mode == 1 ? 0xFu : (T.split_mode == 2 ? ~prevbits : 0u));  // kept spaces that start a word
  const uint32_t out_len = __popc(keep4) + 2u * __popc(keep4 & sp4);
  const uint32_t n_start = __popc(start4);
  const int packed = (int)(out_len | (n_start << 16));
  const int incl = warp_incl_scan(packed, lane);
  const int total = __shfl_sync(kFull, incl, 31);
  if (buffer_empty) {
    if (lane == 0) sm.wstart[0] = 0;
    rs.nw = 1;
  }
  uint32_t o = (uint32_t)rs.nlen + ((uint32_t)(incl - packed) & 0xFFFFu);
  uint8_t* d = sm.nbuf;
  if (keep4 == 0xFu && sp4 == 0u) {  // four plain bytes
    d[o] = (uint8_t)w; d[o + 1] = (uint8_t)(w >> 8); d[o + 2] = (uint8_t)(w >> 16); d[o + 3] = (uint8_t)(w >> 24);
  } else {
    uint32_t wi = (uint32_t)rs.nw + ((uint32_t)(incl - packed) >> 16);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if ((keep4 >> k) & 1u) {
        if ((sp4 >> k) & 1u) {
          if ((start4 >> k) & 1u) sm.wstart[wi++] = (uint16_t)o;
          d[o] = 0xE2; d[o + 1] = 0x96; d[o + 2] = 0x81;
          o += 3;
        } else {
          d[o++] = (uint8_t)(w >> (8 * k));
        }
      }
    }
  }
  // is_prev_space after the window = the last source byte is a space (every unit here is non-empty)
  if (T.remove_extra_ws) {
    const uint32_t n_in = rs.len - pos < (uint32_t)kFastWin ? rs.len - pos : (uint32_t)kFastWin;
    rs.prev_space = (__shfl_sync(kFull, sp4, (n_in - 1) >> 2) >> ((n_in - 1) & 3)) & 1u;
  }
  rs.nlen += total & 0xFFFF;
  rs.nw += total >> 16;
  __syncwarp();
  return true;
}

// ---------------------------------------------------------------------------- word merge
// Fast path: this lane owns word [ws, we) with n <= 32 chars; symbols live in column `lane` of S / PM.
// Returns the alive mask after all merges.
template <bool SMALL, typename SM>
__device__ __forceinline__ uint32_t lane_merge(const SpDev& T, SM& sm, int n, int lane) {
  using P = PMOps<SMALL>;
  uint32_t* S = sm.S + lane;
  typename P::T* PM = sm.PM + lane;
  {
    // initial adjacent pairs, four first probes in flight at a time
    uint32_t left = S[0];
    for (int j0 = 0; j0 + 1 < n; j0 += 4) {
      uint32_t sy[5];
      PairProbe pr[4];
      sy[0] = left;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const bool have = j0 + u + 1 < n;
        sy[u + 1] = have ? S[(j0 + u + 1) * 32] : kSymUnknownFlag;
        pr[u] = pair_probe_begin(T, sy[u], sy[u + 1]);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (j0 + u + 1 < n) PM[(j0 + u) * 32] = P::pack(pair_probe_finish(T, sy[u], sy[u + 1], pr[u]));
      left = sy[4];
    }
  }
  PM[(n - 1) * 32] = P::none();
  uint32_t alive = n >= 32 ? 0xFFFFFFFFu : (1u << n) - 1;
  for (;;) {
    uint32_t best = P::kNone;
    int bj = 0;
    for (uint32_t m = alive; m;) {
      const int j = __ffs(m) - 1;
      m &= m - 1;
      const uint32_t pr = P::prio_at(PM + j * 32);
      if (pr < best) { best = pr; bj = j; }
    }
    if (best == P::kNone) break;
    const uint32_t hi_mask = ~((2u << bj) - 1u);  // bits above bj
    const int rj = __ffs(alive & hi_mask) - 1;
    S[bj * 32] = P::merged(PM[bj * 32]);
    alive &= ~(1u << rj);
    // the two pairs the merge created: both first probes in flight before either is consumed
    const uint32_t above = alive & hi_mask;
    const uint32_t below = alive & ((1u << bj) - 1u);
    const int pj = below ? 31 - __clz(below) : 0;
    const uint32_t sm_ = S[bj * 32];
    const uint32_t sr = above ? S[(__ffs(above) - 1) * 32] : kSymUnknownFlag;
    const uint32_t sl = below ? S[pj * 32] : kSymUnknownFlag;
    const PairProbe pa = pair_probe_begin(T, sm_, sr);
    const PairProbe pb = pair_probe_begin(T, sl, sm_);
    PM[bj * 32] = P::pack(pair_probe_finish(T, sm_, sr, pa));
    if (below) PM[pj * 32] = P::pack(pair_probe_finish(T, sl, sm_, pb));
  }
  return alive;
}

// Cooperative merge of a word of n <= 64 symbols held flat in S[0..n), entirely in registers: lane l owns positions
// l and l + 32 (symbol + the state of the pair that starts there), the alive set is a 64-bit mask every lane holds.
// Per merge: two warp reductions find the best pair (priority, then leftmost), three shuffles bring the merged
// symbol and the two neighbours, and the two new pairs are looked up by their owner lanes at the same time.
// Nothing moves; the survivors are compacted into S[0..ret) at the end.  Same order as coop_merge / lane_merge.
template <bool SMALL>
__device__ __noinline__ int coop_merge64(const SpDev& T, uint32_t* S, int n, int lane) {
  const int p0 = lane, p1 = lane + 32;
  uint32_t sym0 = p0 < n ? S[p0] : kSymUnknownFlag, sym1 = p1 < n ? S[p1] : kSymUnknownFlag;
  const uint32_t nx0 = p0 + 1 < n ? S[p0 + 1] : kSymUnknownFlag, nx1 = p1 + 1 < n ? S[p1 + 1] : kSymUnknownFlag;
  uint2 pm0 = make_uint2(kNoPrio, 0), pm1 = make_uint2(kNoPrio, 0);
  {
    const PairProbe a = pair_probe_begin(T, sym0, nx0), b = pair_probe_begin(T, sym1, nx1);   // both in flight
    if (p0 + 1 < n) pm0 = pair_probe_finish(T, sym0, nx0, a);
    if (p1 + 1 < n) pm1 = pair_probe_finish(T, sym1, nx1, b);
  }
  unsigned long long alive = n >= 64 ? ~0ull : ((1ull << n) - 1ull);
  for (;;) {
    const uint32_t best_prio = __reduce_min_sync(kFull, pm0.x < pm1.x ? pm0.x : pm1.x);
    if (best_prio == kNoPrio) break;
    const uint32_t mine = pm0.x == best_prio ? (uint32_t)p0 : (pm1.x == best_prio ? (uint32_t)p1 : 64u);
    const int bj = (int)__reduce_min_sync(kFull, mine);                 // leftmost pair of the best priority
    const unsigned long long above = alive & ~((2ull << bj) - 1ull);   // bj < 63 here: a pair has a right half
    const int rj = __ffsll((long long)above) - 1;                        // its right half: removed
    alive &= ~(1ull << rj);
    const unsigned long long above2 = above & ~(1ull << rj);
    const unsigned long long below = alive & ((1ull << bj) - 1ull);
    const int nr = above2 ? __ffsll((long long)above2) - 1 : -1;       // next survivor to the right
    const int pj = below ? 63 - __clzll((long long)below) : -1;         // previous survivor
    const uint32_t merged = __shfl_sync(kFull, bj < 32 ? pm0.y : pm1.y, bj & 31);
    const uint32_t sym_nr = __shfl_sync(kFull, (nr & 32) ? sym1 : sym0, nr & 31);
    const uint32_t sym_pj = __shfl_sync(kFull, (pj & 32) ? sym1 : sym0, pj & 31);
    if (lane == (bj & 31)) {
      const uint2 v = nr >= 0 ? pair_lookup(T, merged, sym_nr) : make_uint2(kNoPrio, 0);
      if (bj < 32) { sym0 = merged; pm0 = v; } else { sym1 = merged; pm1 = v; }
    }
    if (lane == (rj & 31)) {                                             // the removed position offers no pair any more
      if (rj < 32) pm0 = make_uint2(kNoPrio, 0); else pm1 = make_uint2(kNoPrio, 0);
    }
    if (pj >= 0 && lane == (pj & 31)) {
      const uint2 v = pair_lookup(T, sym_pj, merged);
      if (pj < 32) pm0 = v; else pm1 = v;
    }
  }
  __syncwarp();
  if ((alive >> p0) & 1ull) S[__popcll(alive & ((1ull << p0) - 1ull))] = sym0;
  if (p1 < 64 && ((alive >> p1) & 1ull)) S[__popcll(alive & ((1ull << p1) - 1ull))] = sym1;
  __syncwarp();
  return __popcll(alive);
}

// Cooperative path: the whole warp merges one word of n (33..1024) chars held flat in S[0..n).
// Returns the final symbol count; S[0..ret) are the final symbols in order.
template <bool SMALL, typename SM>
__device__ int coop_merge(const SpDev& T, SM& sm, int n, int lane) {
  using P = PMOps<SMALL>;
  if (n <= 64) return coop_merge64<SMALL>(T, sm.S, n, lane);
  for (int j = lane; j < n; j += 32)
    sm.PM[j] = j + 1 < n ? P::pack(pair_lookup(T, sm.S[j], sm.S[j + 1])) : P::none();
  __syncwarp();
  for (;;) {
    unsigned long long best = ~0ull;
    for (int j = lane; j + 1 < n; j += 32) {
      const unsigned long long key = ((unsigned long long)P::prio(sm.PM[j]) << 32) | (unsigned)j;
      best = key < best ? key : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long t = __shfl_xor_sync(kFull, best, o);
      best = t < best ? t : best;
    }
    if ((uint32_t)(best >> 32) >= P::kNone) break;
    const int bj = (int)(uint32_t)best;
    const uint32_t merged = P::merged(sm.PM[bj]);
    __syncwarp();
    // remove position bj + 1: shift the tail left by one (tiles in increasing order)
    for (int base = bj + 1; base < n - 1; base += 32) {
      const int k = base + lane;
      uint32_t sv = 0;
      typename P::T pm = P::none();
      const bool act = k < n - 1;
      if (act) { sv = sm.S[k + 1]; pm = sm.PM[k + 1]; }
      __syncwarp();
      if (act) { sm.S[k] = sv; sm.PM[k] = pm; }
      __syncwarp();
    }
    --n;
    // the two pairs the merge created, looked up by two lanes at the same time
    if (lane == 0) {
      sm.S[bj] = merged;
      sm.PM[bj] = bj + 1 < n ? P::pack(pair_lookup(T, merged, sm.S[bj + 1])) : P::none();
    } else if (lane == 1 && bj > 0) {
      sm.PM[bj - 1] = P::pack(pair_lookup(T, sm.S[bj - 1], merged));
    }
    __syncwarp();
  }
  return n;
}

// ---------------------------------------------------------------------------- drain
__device__ __forceinline__ bool is_space_at(const uint8_t* b, int p, int n) {
  return p + 2 < n && b[p] == 0xE2 && b[p + 1] == 0x96 && b[p + 2] == 0x81;
}

// ---------------------------------------------------------------------------- long words
constexpr uint32_t kDeadSym = 0xFFFFFFFFu;
constexpr uint32_t kNoLink = 0xFFFFFFFFu;

// Appends the chars of nbuf[from, to) as symbols to the request's scratch slot.  Returns false when the
// slot's capacity is exceeded.
template <typename SM>
__device__ __noinline__ bool long_append(const SpDev& T, SM& sm, ReqState& rs, int from, int to, int lane) {
  const LongSlot L = long_slot_view(T.long_pool, T.long_cap, rs.long_slot);
  const uint8_t* nb = sm.nbuf;
  bool ok = true;
  for (int base = from; base < to; base += 32) {
    const int p = base + lane;
    const bool lead = p < to && (T.byte_mode || (nb[p] & 0xC0) != 0x80);
    const uint32_t m = __ballot_sync(kFull, lead);
    const uint32_t idx = rs.long_n + __popc(m & ((1u << lane) - 1));
    if (lead) {
      if (idx < T.long_cap) { uint32_t adv; L.sym[idx] = char_sym(T, nb + p, &adv); }
      else ok = false;
    }
    rs.long_n += __popc(m);
  }
  if (to - from >= 3) rs.long_last_sp = nb[to - 3] == 0xE2 && nb[to - 2] == 0x96 && nb[to - 1] == 0x81;
  else if (to > from) rs.long_last_sp = false;
  __syncwarp();
  return !__any_sync(kFull, !ok);
}

// Merges the slot's symbols (bpe_model.cc order: best priority, leftmost on ties) and emits their ids.
__device__ __noinline__ void long_finish(const SpDev& T, ReqState& rs, bool strip_trailing_space, int lane) {
  const LongSlot L = long_slot_view(T.long_pool, T.long_cap, rs.long_slot);
  uint32_t n = rs.long_n;
  if (strip_trailing_space)
    while (n > 0 && L.sym[n - 1] == T.space_sym) --n;
  if (n == 0) return;
  for (uint32_t j = lane; j < n; j += 32) {
    L.next[j] = j + 1 < n ? j + 1 : kNoLink;
    L.prev[j] = j ? j - 1 : kNoLink;
    const uint2 pm = j + 1 < n ? pair_lookup(T, L.sym[j], L.sym[j + 1]) : make_uint2(kNoPrio, 0);
    L.prio[j] = pm.x;
    L.merged[j] = pm.y;
  }
  __syncwarp();
  const uint32_t nb = (n + 31) / 32;
  for (uint32_t b = 0; b < nb; ++b) long_block_min(L, n, b, lane);
  for (;;) {
    unsigned long long best = ~0ull;
    for (uint32_t b = lane; b < nb; b += 32) {
      const unsigned long long k = L.bmin[b];
      best = k < best ? k : best;
    }
    best = warp_min_u64(best);
    if ((uint32_t)(best >> 32) == kNoPrio) break;
    const uint32_t j = (uint32_t)best;
    uint32_t r = 0, p = kNoLink;
    if (lane == 0) {
      r = L.next[j];
      const uint32_t m = L.merged[j];
      const uint32_t nr = L.next[r];
      p = L.prev[j];
      L.sym[j] = m;
      L.next[j] = nr;
      if (nr != kNoLink) L.prev[nr] = j;
      L.prio[r] = kNoPrio;
      L.sym[r] = kDeadSym;
      const uint2 a = nr != kNoLink ? pair_lookup(T, m, L.sym[nr]) : make_uint2(kNoPrio, 0);
      L.prio[j] = a.x;
      L.merged[j] = a.y;
      if (p != kNoLink) {
        const uint2 c = pair_lookup(T, L.sym[p], m);
        L.prio[p] = c.x;
        L.merged[p] = c.y;
      }
    }
    __syncwarp();
    r = __shfl_sync(kFull, r, 0);
    p = __shfl_sync(kFull, p, 0);
    const uint32_t bj = j >> 5, br = r >> 5;
    long_block_min(L, n, bj, lane);
    if (br != bj) long_block_min(L, n, br, lane);
    if (p != kNoLink && (p >> 5) != bj && (p >> 5) != br) long_block_min(L, n, p >> 5, lane);
  }
  // emit the surviving symbols in order
  for (uint32_t base = 0; base < n; base += 32) {
    const uint32_t j = base + lane;
    const uint32_t sym = j < n ? L.sym[j] : kDeadSym;
    const bool alive = sym != kDeadSym;
    int32_t tmp[4];
    bool unk = false;
    int c = alive ? sym_ids(T, sym, tmp, &unk) : 0;
    if (!T.byte_fallback) {
      const uint32_t am = __ballot_sync(kFull, alive);
      const uint32_t um = __ballot_sync(kFull, alive && unk);
      const uint32_t below = am & ((1u << lane) - 1);
      const bool prev = below ? ((um >> (31 - __clz(below))) & 1u) : rs.prev_unk;
      if (alive && unk && prev) c = 0;
      if (am) rs.prev_unk = (um >> (31 - __clz(am))) & 1u;
    }
    const int inc = warp_incl_scan(c, lane);
    int64_t o = rs.n_out + (inc - c);
    for (int k = 0; k < c; ++k) put_id(rs, o++, tmp[k]);
    rs.n_out += __shfl_sync(kFull, inc, 31);
  }
  rs.trailing_bare = 0;
  __syncwarp();
}

// Long mode: nbuf continues the slot's word.  Appends up to the first word boundary (or everything),
// finishes the word when its end is known, and returns to the normal mode with the rest of nbuf.
template <typename SM>
__device__ __noinline__ void long_consume(const SpDev& T, SM& sm, ReqState& rs, bool final, int lane) {
  const uint8_t* nb = sm.nbuf;
  const int nlen = rs.nlen;
  int cut = nlen;
  if (T.split_mode != 0) {
    for (int base = 0; base < nlen && cut == nlen; base += 32) {
      const int p = base + lane;
      bool st = false;
      if (p < nlen && is_space_at(nb, p, nlen)) {
        const bool prev_sp = p >= 3 ? is_space_at(nb, p - 3, nlen) : (p == 0 && rs.long_last_sp);
        st = T.split_mode == 1 || !prev_sp;
      }
      const uint32_t m = __ballot_sync(kFull, st);
      if (m) cut = base + __ffs(m) - 1;
    }
  }
  if (!long_append(T, sm, rs, 0, cut, lane)) {
    rs.too_long = true;
    long_slot_release(T.long_locks, rs.long_slot, lane);
    rs.long_mode = false;
    return;
  }
  if (cut < nlen || final) {
    long_finish(T, rs, final && cut == nlen && T.remove_extra_ws, lane);
    long_slot_release(T.long_locks, rs.long_slot, lane);
    rs.long_mode = false;
    const int tl = nlen - cut;
    if (cut > 0) {
      for (int base = 0; base < tl; base += 32) {
        const int k = base + lane;
        uint8_t c = 0;
        if (k < tl) c = sm.nbuf[cut + k];
        __syncwarp();
        if (k < tl) sm.nbuf[k] = c;
        __syncwarp();
      }
    }
    rs.nlen = tl;
  } else {
    rs.nlen = 0;
  }
  rs.rescan = true;
  rs.ascii = false;
  rs.nw = 0;
  __syncwarp();
}

// Switches to long mode: nbuf holds exactly one incomplete word (the tail a drain kept).
template <typename SM>
__device__ __noinline__ bool long_enter(const SpDev& T, SM& sm, ReqState& rs, int lane) {
  if (T.long_slots <= 0) return false;
  rs.long_slot = long_slot_acquire(T.long_locks, T.long_slots, lane);
  rs.long_n = 0;
  rs.long_last_sp = false;
  rs.long_mode = true;
  if (!long_append(T, sm, rs, 0, rs.nlen, lane)) {
    long_slot_release(T.long_locks, rs.long_slot, lane);
    rs.long_mode = false;
    return false;
  }
  rs.nlen = 0;
  rs.rescan = true;
  rs.ascii = false;
  rs.nw = 0;
  return true;
}

#ifdef XLLM_MEMO_STATS
__device__ unsigned long long g_memo_stats[8];
#endif
struct MemoRef {
  uint8_t* table;
  uint32_t mask;
};

// ---------------------------------------------------------------------------- Unigram
// unigram_model.cc Model::EncodeOptimized for ONE word w[0, len) whose best path starts from *score (the best-path
// score at the word start, carried as a float across words exactly as upstream's best_path_ends_at[].best_path_score).
// No NORMAL piece spans a word start (split_mode 1/2, checked by the loader), so every path of the sentence passes
// through it and the sentence's Viterbi factors into per-word ones — but each word has to start from the running
// float score, because candidates are formed as double(piece score) + double(float score so far) and stored back
// as float: rounding makes the winner depend on everything before the word.
// The warp walks the word's end positions; lane L-1 proposes the piece of L bytes that ends there (one probe of the
// bytes -> id table), the candidates are then folded in upstream's order (ascending start = descending length,
// strict '>' against the stored float), a char no piece covers costs unk_score.  best[] lives in S[], the back
// links in PM[].  Returns the symbol count; S[0..n) = kResolvedFlag | piece id, or kSymUnknownFlag | code point.
constexpr int kUniMaxWord = 511;  // bytes per word (best[] has kCoopMaxSym entries)

// (parent node, byte) -> child node and its piece id (-1: a proper prefix only); false: no piece continues this way
__device__ __forceinline__ bool uni_trie_step(const SpDev& T, uint32_t parent, uint32_t byte, uint32_t* child,
                                              int32_t* piece) {
  uint32_t h = (parent * 256u + byte) * 0x9E3779B1u;  // sp_trie_slot (sp_model.cc)
  h ^= h >> 15;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  uint32_t slot = h & T.utrie_mask;
  for (;;) {
    const uint4 e = __ldg(T.utrie + slot);
    if (e.x == parent && e.y == byte) { *child = e.z; *piece = (int32_t)e.w; return true; }
    if (e.x == 0xFFFFFFFFu) return false;
    slot = (slot + 1) & T.utrie_mask;
  }
}

template <typename SM>
__device__ int unigram_backtrack(SM& sm, const uint8_t* w, int len, int lane);
template <typename SM>
__device__ int unigram_word_slow(const SpDev& T, SM& sm, const uint8_t* w, int len, float* score, int lane);

// The same lattice built the way upstream builds it — from the START positions: 32 starts at a time, every lane walks
// the piece trie from its start until no piece continues (a few dependent L2 probes, all lanes in parallel) and
// lists what it found; then the starts are folded in order (as upstream's outer loop), lane k applying the k-th
// piece of the current start to best[start + length] — distinct ends, so no conflicts inside a start.
// Falls back to unigram_word_slow when one start has more than kUniMaxMatch pieces.
template <typename SM>
__device__ int unigram_word(const SpDev& T, SM& sm, const uint8_t* w, int len, float* score, int lane) {
  float* best = reinterpret_cast<float*>(sm.S);
  uint32_t* back = reinterpret_cast<uint32_t*>(sm.PM);  // 0 = no path ends here yet
  for (int e = lane; e <= len; e += 32) back[e] = 0;
  if (lane == 0) best[0] = *score;
  __syncwarp();
  for (int s0 = 0; s0 < len; s0 += 32) {
    // ---- walk the trie from every start of this block
    const int s = s0 + lane;
    const bool is_start = s < len && (w[s] & 0xC0) != 0x80;
    int cnt = 0;
    bool overflow = false;
    if (is_start) {
      const uint8_t b0 = w[s];
      int clen = b0 < 0x80 ? 1 : (b0 < 0xE0 ? 2 : (b0 < 0xF0 ? 3 : 4));
      if (clen > len - s) clen = len - s;
      const int max_l = (int)T.max_piece_len < len - s ? (int)T.max_piece_len : len - s;
      uint32_t node = 0;
      bool has_single = false;
      for (int L = 1; L <= max_l; ++L) {
        int32_t piece;
        if (!uni_trie_step(T, node, w[s + L - 1], &node, &piece)) break;
        if (piece >= 0) {
          if (cnt < kUniMaxMatch) sm.mlist[lane * kUniMaxMatch + cnt] = ((uint32_t)L << 24) | (uint32_t)piece;
          else overflow = true;
          ++cnt;
          has_single |= L == clen;
        }
      }
      if (!has_single) {  // no piece is exactly this char: the unknown candidate
        if (cnt < kUniMaxMatch) sm.mlist[lane * kUniMaxMatch + cnt] = ((uint32_t)clen << 24) | 0xFFFFFFu;
        else overflow = true;
        ++cnt;
      }
    }
    if (__any_sync(kFull, overflow)) return unigram_word_slow(T, sm, w, len, score, lane);
    __syncwarp();
    // ---- fold the starts in order
    uint32_t starts = __ballot_sync(kFull, is_start);
    while (starts) {
      const int b = __ffs(starts) - 1;
      starts &= starts - 1;
      const int sb = s0 + b;
      const int nb_ = __shfl_sync(kFull, cnt, b);
      const float base = best[sb];
      if (lane < nb_) {
        const uint32_t m = sm.mlist[b * kUniMaxMatch + lane];
        const int L = (int)(m >> 24);
        const uint32_t id = m & 0xFFFFFFu;
        const int e = sb + L;
        const double cand = id == 0xFFFFFFu ? (double)(T.unk_score + base)  // float + float upstream
                                            : (double)__ldg(T.piece_score + id) + (double)base;
        if (back[e] == 0 || cand > (double)best[e]) {
          best[e] = (float)cand;
          back[e] = m;
        }
      }
      __syncwarp();
    }
  }
  const float end_score = best[len];
  __syncwarp();
  const int n = unigram_backtrack(sm, w, len, lane);
  *score = end_score;
  __syncwarp();
  return n;
}

// back[] -> S[0..n): kResolvedFlag | piece id, or kSymUnknownFlag | code point
template <typename SM>
__device__ int unigram_backtrack(SM& sm, const uint8_t* w, int len, int lane) {
  const uint32_t* back = reinterpret_cast<const uint32_t*>(sm.PM);
  int n = 0;
  for (int e = len; e > 0; e -= (int)(back[e] >> 24)) ++n;
  __syncwarp();
  if (lane == 0) {
    int k = n;
    for (int e = len; e > 0;) {
      const uint32_t link = back[e];
      const int L = (int)(link >> 24);
      uint32_t sym;
      if ((link & 0xFFFFFFu) != 0xFFFFFFu) {
        sym = kResolvedFlag | (link & 0xFFFFFFu);
      } else {
        const uint8_t* p = w + e - L;
        const uint32_t b0 = p[0];
        uint32_t cp = b0;
        if (L == 2) cp = ((b0 & 0x1F) << 6) | (p[1] & 0x3F);
        else if (L == 3) cp = ((b0 & 0x0F) << 12) | ((p[1] & 0x3Fu) << 6) | (p[2] & 0x3F);
        else if (L == 4) cp = ((b0 & 0x07) << 18) | ((p[1] & 0x3Fu) << 12) | ((p[2] & 0x3Fu) << 6) | (p[3] & 0x3F);
        sym = kSymUnknownFlag | cp;
      }
      sm.S[--k] = sym;
      e -= L;
    }
  }
  __syncwarp();
  return n;
}

// The per-END-position form (kept as the fallback): lane L-1 proposes the piece of L bytes that ends at e.
template <typename SM>
__device__ int unigram_word_slow(const SpDev& T, SM& sm, const uint8_t* w, int len, float* score, int lane) {
  float* best = reinterpret_cast<float*>(sm.S);
  uint32_t* back = reinterpret_cast<uint32_t*>(sm.PM);  // id (24 bits, 0xFFFFFF = unknown char) | length << 24
  static_assert(sizeof(sm.S) >= 4 * (kUniMaxWord + 1) && sizeof(sm.PM) >= 4 * (kUniMaxWord + 1), "lattice scratch");
  if (lane == 0) best[0] = *score;
  __syncwarp();
  const int passes = ((int)T.max_piece_len + 31) / 32;
  for (int e = 1; e <= len; ++e) {
    if (e < len && (w[e] & 0xC0) == 0x80) continue;  // not a char boundary
    int cs = e - 1;
    while (cs > 0 && (w[cs] & 0xC0) == 0x80) --cs;
    const int clen = e - cs;  // bytes of the char that ends at e
    float best_f = 0.f;
    uint32_t best_link = 0;
    bool first = true;
    for (int pass = passes - 1; pass >= 0; --pass) {  // longest pieces (earliest starts) first
      const int L = pass * 32 + lane + 1;
      const int s = e - L;
      int32_t id = -1;
      if (L <= (int)T.max_piece_len && s >= 0 && (w[s] & 0xC0) != 0x80) id = hf_vocab_lookup(T, w + s, L);
      const bool unk = id < 0 && L == clen;  // no piece is exactly this char: the unknown candidate of its start
      double cand = 0.0;
      if (id >= 0) cand = (double)__ldg(T.piece_score + id) + (double)best[s];
      else if (unk) cand = (double)(T.unk_score + best[s]);  // float + float upstream
      uint32_t m = __ballot_sync(kFull, id >= 0 || unk);
      while (m) {
        const int src = 31 - __clz(m);
        m &= ~(1u << src);
        const double c = __shfl_sync(kFull, cand, src);
        const int32_t cid = __shfl_sync(kFull, id, src);
        if (first || c > (double)best_f) {
          best_f = (float)c;
          best_link = ((uint32_t)(pass * 32 + src + 1) << 24) | (cid >= 0 ? (uint32_t)cid : 0xFFFFFFu);
          first = false;
        }
      }
    }
    if (lane == 0) { best[e] = best_f; back[e] = best_link; }
    __syncwarp();
  }
  const float end_score = best[len];
  __syncwarp();
  const int n = unigram_backtrack(sm, w, len, lane);
  *score = end_score;
  __syncwarp();
  return n;
}

// ---------------------------------------------------------------------------- express path
// One step tokenises one 512-byte source window straight from the loaded bytes: no normalized-text buffer, no word list,
// no symbol columns for words the memo knows.  It runs only in the BOUNDARY state — nbuf is empty, or holds exactly
// the one U+2581 (dummy prefix / kept space) that leads the next word — and only for models with split_mode 1 and
// remove_extra_whitespaces (every kept space starts a word, runs of spaces collapse), on windows that pass the
// fast path's own test (every byte a simple or space-like ASCII byte followed by an ASCII byte), so the normalizer's
// output is known without writing it:  word = maximal run of non-space bytes, led by U+2581 iff a kept space or the
// dummy prefix precedes it.  Lane k takes the k-th and (k + 32)-th COMPLETE words of the window (their ends are in the window or at
// the end of the text), reads their <= 15 bytes from the window staged in shared memory, builds the memo key and probes;
// a miss is merged in the lane's symbol column exactly as a drain round would and inserted.  Ids are written from
// the memo payload.  The step consumes up to the start of the first word it did not take and leaves the state a
// drain would have left.  Anything it cannot do exactly (a word over 15 bytes, an unknown symbol, a word of more
// ids than a memo payload holds) returns 0 with nothing changed, and the window goes through the buffer path.
// Diagnostics build (-DXLLM_EXP_STATS): event counters, and lane 0's clock64() split of the steps that resolve words
// into three phases (window: step start to the classification vote, the first use of the loaded text; probe: to the
// ballot that first depends on the memo loads; emit: to after the id stores), summed per warp and added at the end.
#ifdef XLLM_EXP_STATS
constexpr int kExpStats = 32;
enum : int { kExpStatTimed = 16, kExpStatCycWindow = 17, kExpStatCycProbe = 18, kExpStatCycEmit = 19 };
__device__ unsigned long long g_exp_stats[kExpStats];
#define EXP_STAT(i) do { if (lane == 0) atomicAdd(&g_exp_stats[i], 1ull); } while (0)
#define EXP_CLOCK(t) (t = clock64())
#else
#define EXP_STAT(i) do { } while (0)
#define EXP_CLOCK(t) do { } while (0)
#endif

// Runs express steps from source offset pos for as long as they apply; returns the offset reached and sets *failed
// when it stopped in front of a window it cannot do (the caller sends that window through the buffer path).
// Windows are 16-byte ALIGNED: the step loads the 32 aligned 16-byte units from the one that holds pos, turns the bytes
// in front of pos (and past the end of the text) into spaces, and never consumes byte 511 of a window unless the text
// ends inside it — so every consumed byte has its successor inside the window, where it was checked to be ASCII.
struct ExpReq {
  const uint8_t* src;
  uint32_t len;
  int32_t* out;
  int64_t cap;     // ids that fit the row
  int64_t n_out;   // ids produced so far (may exceed cap)
  bool P;          // a U+2581 is pending in front of the next word (dummy prefix / kept space)
  bool S;          // the normalizer's is_prev_space
  bool U;          // the last emitted symbol was unknown (matters with byte_fallback off only)
};
// per warp: symbol columns for the words the memo does not know yet, the window's text and its words' {start, end}
constexpr int kExpWords = 64;        // words an express step resolves: lane k takes words k and k + 32
template <bool SMALL>
struct ExpSmemT {
  uint32_t S[kMaxSym * 32];
  typename PMOps<SMALL>::T PM[kMaxSym * 32];
  uint4 txt[kExpWin / 16 + 1];       // the window (16 bytes per lane) + 16 bytes a word's key read may touch past it
  uint16_t ex[2 * (kExpWords + 2)];  // {start, end} of words 0 .. kExpWords - 1, and the start of word kExpWords
};
constexpr int kExpLongWords = 4;     // express_run: long words a request may put through the cooperative path ...
constexpr int kExpLongEvery = 512;   // ... at a density above one per this many bytes before it is handed over
// what the buffer-path kernel needs to take a request over where the express kernel stopped
struct ExpResume {
  uint32_t pos;      // source bytes consumed
  uint32_t flags;    // bit 0: P, bit 1: S, bit 2: U (ExpReq)
  long long n_out;
};

// The outcome of express_long_word, returned by value (no address-taken locals in the express loop)
struct ExpLongWord {
  uint32_t end;      // offset of the byte after the word (done only)
  int32_t n_out;     // ids produced so far (unchanged unless done)
  bool done;
  bool unk;          // the last emitted symbol was unknown
};

// A word the lane path does not take — more than 15 bytes, or one whose ids do not fit a memo payload (an unknown
// symbol, byte fallback, more than 7 / 4 ids) — merged by the whole warp in the flat symbol scratch, as the buffer
// path's cooperative branch does.  v0 = offset of its first byte.  Finds the word's end (a space / space-like byte or
// the end of the text), checking that every byte is a simple ASCII byte; not done (nothing emitted) when it is not, or
// when the word has more chars than the scratch holds.
template <bool SMALL, typename SM>
__device__ __noinline__ ExpLongWord express_long_word(const SpDev& T, SM& sm, const uint32_t* base, uint32_t nwords,
                                                      uint32_t vlen, uint32_t v0, bool lead, int32_t* out, int32_t cap,
                                                      int32_t n_out, bool prev_unk, int lane) {
  const ExpLongWord not_done{0u, n_out, false, prev_unk};
  // --- the end of the word
  uint32_t end = 0;
  bool found = false;
  for (uint32_t wb = v0 & ~3u; !found; wb += (uint32_t)kFastWin) {
    if (wb - (v0 & ~3u) > (uint32_t)kCoopMaxSym) return not_done;   // longer than the scratch
    const uint32_t i = (wb >> 2) + (uint32_t)lane;
    uint32_t w = i < nwords ? __ldg(base + i) : 0x20202020u;
    const uint32_t b0 = wb + 4u * lane;                            // offset of the lane's first byte
    uint32_t sp4 = 0, bad4 = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t bk = (w >> (8 * k)) & 0xFFu;
      const uint32_t at = b0 + k;
      if (at < v0) continue;                                       // in front of the word
      if (at >= vlen) { sp4 |= 1u << k; continue; }                // past the end of the text: ends the word
      if (bk >= 0x80u) { bad4 |= 1u << k; continue; }
      const bool spl = bk == 0x20u || ((T.spacelike_ascii[(bk >> 5) & 3] >> (bk & 31)) & 1u);
      const bool simple = (T.simple_ascii[(bk >> 5) & 3] >> (bk & 31)) & 1u;
      if (spl && (bk != 0x20u || simple)) sp4 |= 1u << k;
      else if (!simple) bad4 |= 1u << k;
    }
    const uint32_t spm = __ballot_sync(kFull, sp4 != 0u), badm = __ballot_sync(kFull, bad4 != 0u);
    if (spm) {
      const int L = __ffs(spm) - 1;
      const uint32_t sL = __shfl_sync(kFull, sp4, L), bL = __shfl_sync(kFull, bad4, L);
      const int k = __ffs(sL) - 1;
      if ((badm & ((1u << L) - 1u)) || (bL & ((1u << k) - 1u))) return not_done;   // a byte the fast rules do not cover
      end = wb + 4u * L + k;
      found = true;
    } else if (badm) {
      return not_done;
    }
  }
  const int nbytes = (int)(end - v0);
  const int nsym = nbytes + (lead ? 1 : 0);
  if (nbytes < 1 || nsym > kCoopMaxSym) return not_done;
  // --- symbols, merge, ids
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(base) + v0;
  __syncwarp();   // the lanes' own merges of this step (their columns of S / PM) are done before S is rewritten flat
  if (lead && lane == 0) sm.S[0] = T.space_sym;
  for (int i = lane; i < nbytes; i += 32) sm.S[i + (lead ? 1 : 0)] = __ldg(T.ascii_sym + __ldg(bytes + i));
  __syncwarp();
  const int n = coop_merge<SMALL>(T, sm, nsym, lane);
  for (int b = 0; b < n; b += 32) {
    const int j = b + lane;
    int32_t tmp[4];
    bool unk = false;
    int c = 0;
    if (j < n) c = sym_ids(T, sm.S[j], tmp, &unk);
    if (!T.byte_fallback) {   // consecutive unknown symbols give one <unk>
      const uint32_t um = __ballot_sync(kFull, j < n && unk);
      const bool prev = lane == 0 ? prev_unk : ((um >> (lane - 1)) & 1u);
      if (unk && prev) c = 0;
      const int lastl = (n - b) >= 32 ? 31 : (n - b - 1);
      prev_unk = (um >> lastl) & 1u;
    }
    const int inc = warp_incl_scan(c, lane);
    int32_t o = n_out + (inc - c);
    for (int k = 0; k < c; ++k, ++o)
      if (o < cap) out[o] = tmp[k];
    n_out += __shfl_sync(kFull, inc, 31);
  }
  if (T.byte_fallback) prev_unk = false;
  __syncwarp();
  return ExpLongWord{end, n_out, true, prev_unk};
}

// Bytes of x (bytes 4i .. 4i + 3 of the lane's 16) outside [lo, hi) become spaces.
__device__ __forceinline__ uint32_t exp_blank(uint32_t x, int i, int lo, int hi) {
  const int a = min(max(lo - 4 * i, 0), 4), b = min(max(hi - 4 * i, 0), 4);
  const uint32_t below_b = b >= 4 ? 0xFFFFFFFFu : (1u << (8 * b)) - 1u, below_a = a >= 4 ? 0xFFFFFFFFu : (1u << (8 * a)) - 1u;
  const uint32_t keep = below_b & ~below_a;
  return (x & keep) | (0x20202020u & ~keep);
}
// 0x80 in every space byte of x -> one bit per byte
__device__ __forceinline__ uint32_t exp_space4(uint32_t x) {
  x ^= 0x20202020u;
  const uint32_t z = ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);
  return (((z >> 7) * 0x01020408u) >> 24) & 0xFu;
}
// The memo key (memo_key's layout) of the n <= 15 bytes of the window's text from offset s.
__device__ __forceinline__ U128 exp_word_key(const uint4* txt, uint32_t s, int n, bool lead) {
  const uint2* t8 = reinterpret_cast<const uint2*>(txt) + (s >> 3);
  const uint2 u0 = t8[0], u1 = t8[1], u2 = t8[2];
  const bool odd = (s & 4u) != 0u;
  const uint32_t bsh = (s & 3u) * 8u;
  const uint32_t t0 = odd ? u0.y : u0.x, t1 = odd ? u1.x : u0.y, t2 = odd ? u1.y : u1.x, t3 = odd ? u2.x : u1.y,
                 t4 = odd ? u2.y : u2.x;
  unsigned long long lo = (unsigned long long)__funnelshift_r(t0, t1, bsh) | ((unsigned long long)__funnelshift_r(t1, t2, bsh) << 32);
  unsigned long long hi = (unsigned long long)__funnelshift_r(t2, t3, bsh) | ((unsigned long long)__funnelshift_r(t3, t4, bsh) << 32);
  if (n < 8) { lo &= (1ull << (8 * n)) - 1ull; hi = 0ull; }
  else hi &= (1ull << (8 * (n - 8))) - 1ull;
  return U128{(lo << 8) | (unsigned long long)((lead ? 0x80u : 0u) | (uint32_t)n), (hi << 8) | (lo >> 56)};
}
// The memo probe's second half: compare the first way loaded by the caller, load the second way when the first holds
// another word.  Returns hit (a key match with ids); val holds the payload of the way that matched.  Both ways are
// loaded with ld_b128_cached: the hot words' slots stay in the SM's L1, which takes the L2 round trip off most
// probes, the longest link of a step.  A slot read before another SM's insert reaches it reads as a miss: the lane
// merges the word, and its insert's CAS, which goes to L2, finds the key there.
template <bool SMALL>
__device__ __forceinline__ bool exp_probe_finish(MemoRef memo, U128 key, uint32_t slot, U128 k, U128& val) {
  if (k.lo == key.lo && k.hi == key.hi) return MemoIds<SMALL>::valid(val);
  if ((k.lo | k.hi) == 0) return false;
  const uint8_t* e = memo.table + (size_t)(slot ^ 1u) * 32;
  const U128 k2 = ld_b128_cached(e);
  val = ld_b128_cached(e + 16);
  return k2.lo == key.lo && k2.hi == key.hi && MemoIds<SMALL>::valid(val);
}
// A word's ids from its memo payload at out[o ..]; c1 / c2: some lane of the warp has a word of >= 2 / >= 4 ids.
template <bool SMALL>
__device__ __forceinline__ void exp_store(int32_t* out, U128 val, int cnt, int o, bool c1, bool c2, bool fits,
                                          int32_t cap) {
  if (fits) {      // the whole step fits the row (always, but for a truncating ids_stride)
    if (cnt >= 1) out[o] = (int32_t)MemoIds<SMALL>::id(val, 0);
    if (c1 || c2) {
      if (cnt >= 2) out[o + 1] = (int32_t)MemoIds<SMALL>::id(val, 1);
      if (cnt >= 3) out[o + 2] = (int32_t)MemoIds<SMALL>::id(val, 2);
      if (c2) {
#pragma unroll
        for (int q = 3; q < MemoIds<SMALL>::kMax; ++q)
          if (q < cnt) out[o + q] = (int32_t)MemoIds<SMALL>::id(val, q);
      }
    }
  } else {
#pragma unroll
    for (int q = 0; q < MemoIds<SMALL>::kMax; ++q)
      if (q < cnt && o + q < cap) out[o + q] = (int32_t)MemoIds<SMALL>::id(val, q);
  }
}

template <bool SMALL, bool MEMO, typename SM>
__device__ __forceinline__ uint32_t express_run(const SpDev& T, SM& sm, ExpReq& rs, uint32_t pos, int lane,
                                                MemoRef memo, bool* failed) {
  // 32-bit coordinates: v = byte offset from the 16-byte-aligned address at or below the request's first byte
  const uint32_t A = (uint32_t)(reinterpret_cast<uintptr_t>(rs.src) & 15u);
  const uint32_t* const base = reinterpret_cast<const uint32_t*>(rs.src - A);
  const uint4* const base16 = reinterpret_cast<const uint4*>(rs.src - A);
  const uint32_t vlen = rs.len + A;                 // end of the text
  const uint32_t nwords = (vlen + 3u) >> 2;         // aligned 4-byte words that hold text (express_long_word)
  const uint32_t nunits = (vlen + 15u) >> 4;        // aligned 16-byte units that hold text
  bool P = rs.P;
  bool S = rs.S;
  bool U = rs.U;
  int n_long = 0;             // long words this request sent through the cooperative path
  uint16_t* const ex = sm.ex;
  const uint32_t* const ex2 = reinterpret_cast<const uint32_t*>(sm.ex);   // {start, end} of word k as one u32
  int32_t* const out = rs.out;
  const int32_t cap = rs.cap > 0x7fffffffll ? 0x7fffffff : (int32_t)rs.cap;
  int32_t n_out = (int32_t)rs.n_out;
  const uint32_t lt = (1u << lane) - 1u;
  auto load_window = [&](uint32_t at) {             // the 32 aligned 16-byte units from the one that holds byte `at`
    const uint32_t i = (at >> 4) + (uint32_t)lane;
    return i < nunits ? __ldg(base16 + i) : make_uint4(0x20202020u, 0x20202020u, 0x20202020u, 0x20202020u);
  };
  uint32_t v = pos + A;
  uint4 w = load_window(v);
  *failed = false;
#ifdef XLLM_EXP_STATS
  unsigned long long t_step = 0, t_vote = 0, t_probe = 0, cyc_window = 0, cyc_probe = 0, cyc_emit = 0, n_timed = 0;
#endif
  for (;;) {
    EXP_CLOCK(t_step);
    const uint32_t skip = v & 15u;
    const uint32_t wb = v - skip;                                  // the window's first (aligned) byte
    const bool at_end = wb + (uint32_t)kExpWin >= vlen;            // the text ends inside this window
    if ((skip != 0u && lane == 0) || at_end) {                     // bytes in front of the position / past the end: spaces
      const int lo = lane == 0 ? (int)skip : 0;
      const int hi = at_end ? (int)(vlen - wb) - 16 * lane : 16;
      w = make_uint4(exp_blank(w.x, 0, lo, hi), exp_blank(w.y, 1, lo, hi), exp_blank(w.z, 2, lo, hi),
                     exp_blank(w.w, 3, lo, hi));
    }
    {
      // every byte a simple ASCII byte (then it is its own unit, given an ASCII successor) or a space-like one
      bool ok = ((w.x | w.y | w.z | w.w) & 0x80808080u) == 0u;
      bool fast_ok = false;
      if (T.printable_simple)
        fast_ok = (((w.x | 0x80808080u) - 0x20202020u) & ((w.y | 0x80808080u) - 0x20202020u) &
                   ((w.z | 0x80808080u) - 0x20202020u) & ((w.w | 0x80808080u) - 0x20202020u) & 0x80808080u) ==
                      0x80808080u &&                                                            // every byte >= 0x20
                  (((w.x + 0x01010101u) | (w.y + 0x01010101u) | (w.z + 0x01010101u) | (w.w + 0x01010101u)) &
                   0x80808080u) == 0u;                                                          // every byte <= 0x7E
      if (!__all_sync(kFull, ok && fast_ok)) {
        uint32_t q[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          uint32_t& part = q[k >> 2];
          const uint32_t bk = (part >> (8 * (k & 3))) & 0xFFu;
          const bool spl = (T.spacelike_ascii[(bk >> 5) & 3] >> (bk & 31)) & 1u;
          ok = ok && (spl || ((T.simple_ascii[(bk >> 5) & 3] >> (bk & 31)) & 1u));
          if (spl) part = (part & ~(0xFFu << (8 * (k & 3)))) | (0x20u << (8 * (k & 3)));
        }
        if (!__all_sync(kFull, ok)) { EXP_STAT(4); *failed = true; break; }
        w = make_uint4(q[0], q[1], q[2], q[3]);
      }
    }
    EXP_CLOCK(t_vote);
    // non-space bytes of the lane's 16 bytes; word starts / ends from the two neighbouring bytes
    const uint32_t ns16 = ~(exp_space4(w.x) | (exp_space4(w.y) << 4) | (exp_space4(w.z) << 8) | (exp_space4(w.w) << 12)) &
                          0xFFFFu;
    sm.txt[lane] = w;                                              // the words' bytes are read from here
    uint32_t prev_ns = (__shfl_up_sync(kFull, ns16, 1) >> 15) & 1u;
    uint32_t next_ns = __shfl_down_sync(kFull, ns16, 1) & 1u;
    if (lane == 0) prev_ns = 0u;
    if (lane == 31) next_ns = at_end ? 0u : 1u;                    // unknown successor: the word is not complete
    if (!P && !S) {                                                // would continue a word that is not in the buffer
      if ((__shfl_sync(kFull, ns16, 0) >> skip) & 1u) { EXP_STAT(5); *failed = true; break; }
    }
    const uint32_t st16 = ns16 & ~((ns16 << 1) | prev_ns) & 0xFFFFu;
    const uint32_t en16 = ns16 & ~((ns16 >> 1) | (next_ns << 15)) & 0xFFFFu;
    // starts per lane: 0..8 (four bits) -> four ballots give every lane the index of its first start
    const uint32_t cs = __popc(st16);
    const uint32_t b0 = __ballot_sync(kFull, cs & 1u), b1 = __ballot_sync(kFull, cs & 2u);
    const uint32_t b2 = __ballot_sync(kFull, cs & 4u), b3 = __ballot_sync(kFull, cs & 8u);
    const uint32_t last_ns = __ballot_sync(kFull, (ns16 & 0x8000u) != 0u) >> 31;
    const int nstart = __popc(b0) + 2 * __popc(b1) + 4 * __popc(b2) + 8 * __popc(b3);
    const int nend = nstart - (int)(at_end ? 0u : last_ns);       // an unfinished word at the end of the window
    int take = nend < kExpWords ? nend : kExpWords;                // complete words this step resolves
    uint32_t cons = at_end ? vlen - wb : (uint32_t)kExpWin - 1u;   // window bytes consumed (counted from wb)
    bool S2 = true;
    uint4 w_next = make_uint4(0u, 0u, 0u, 0u);
    // a word the lane path does not take, at window offset s0, through the cooperative path; false: the run stops
    // (the text is done, or the request is handed over at the word)
    auto long_word = [&](uint32_t s0) -> bool {
      // a text dense in long words (natural text: one in ~100 bytes) is better off in the buffer-path kernel, which
      // merges words of up to 32 symbols 32 at a time in lane columns: after kExpLongWords of them at more than one
      // per kExpLongEvery bytes the rest of the request is handed over
      ++n_long;
      const bool dense = n_long > kExpLongWords && (uint32_t)n_long * (uint32_t)kExpLongEvery > wb + s0 - A;
      ExpLongWord r{0u, n_out, false, U};
      if (!dense) r = express_long_word<SMALL>(T, sm, base, nwords, vlen, wb + s0, P || (!S && s0 > skip), out, cap,
                                              n_out, U, lane);
      n_out = r.n_out;
      U = r.unk;
      if (!r.done) {
        if (s0 > skip) {                           // hand over at the word, with the spaces in front of it consumed
          P = P || !S;
          S = true;
          v = wb + s0;
        }
        *failed = true;
        return false;
      }
      P = false;                                   // the byte before r.end is the word's last: nothing pending
      S = false;
      v = r.end;
      if (v >= vlen) return false;
      w = load_window(v);
      return true;
    };
    if (nstart > 0) {
      {
        uint32_t k = __popc(b0 & lt) + 2 * __popc(b1 & lt) + 4 * __popc(b2 & lt) + 8 * __popc(b3 & lt);
        uint32_t e = k - (prev_ns & ns16 & 1u);    // words that ended before this lane = started - the one still open
        for (uint32_t m = st16; m && k <= (uint32_t)kExpWords; m &= m - 1u, ++k)
          ex[2u * k] = (uint16_t)(16 * lane + __ffs(m) - 1);
        for (uint32_t m = en16; m && e < (uint32_t)kExpWords; m &= m - 1u, ++e)
          ex[2u * e + 1u] = (uint16_t)(16 * lane + __ffs(m) - 1);
      }
      __syncwarp();
      const bool inA = lane < take, inB = lane + 32 < take;
      const uint32_t seA = ex2[inA ? lane : 0], seB = ex2[inB ? lane + 32 : 0];
      const uint32_t sA = seA & 0xFFFFu, sB = seB & 0xFFFFu;
      const int nA = (int)(seA >> 16) - (int)sA + 1, nB = (int)(seB >> 16) - (int)sB + 1;
      // the lane path takes words of up to 15 bytes: stop in front of the first longer one (in text order)
      const uint32_t lmA = __ballot_sync(kFull, inA && nA > kMemoMaxKeyBytes);
      const uint32_t lmB = __ballot_sync(kFull, inB && nB > kMemoMaxKeyBytes);
      if (lmA) take = __ffs(lmA) - 1;
      else if (lmB) take = 32 + __ffs(lmB) - 1;
      if (take == 0) {
        // the first word is long, or not finished inside this window
        const uint32_t s0 = ex[0];
        if (!lmA && s0 > skip) {
          cons = s0;                               // only spaces in front of it: take those, the word starts the next window
          w_next = load_window(wb + cons);
        } else {
          if (long_word(s0)) { EXP_STAT(6); continue; }
          EXP_STAT(7);
          break;
        }
      } else {
      const bool activeA = lane < take, activeB = lane + 32 < take;
      if (take < nstart) cons = ex[2 * take];      // stop in front of the first word not taken
      // --- the words' memo keys: {lead U+2581, length} byte + the word's bytes (all a miss needs later, too)
      const bool leadA = lane > 0 || P || (!S && sA > skip);       // word k + 32 always follows a kept space
      const U128 keyA = exp_word_key(sm.txt, sA, nA, leadA), keyB = exp_word_key(sm.txt, sB, nB, true);
      // --- memo: both words' first ways in flight before either is compared
      bool hitA = false, hitB = false;
      U128 valA{0ull, 0ull}, valB{0ull, 0ull};
      if constexpr (MEMO) {
        const uint32_t slotA = memo_slot(keyA, memo.mask), slotB = memo_slot(keyB, memo.mask);
        U128 kA{0ull, 0ull}, kB{0ull, 0ull};
        if (activeA) {
          kA = ld_b128_cached(memo.table + (size_t)slotA * 32);
          valA = ld_b128_cached(memo.table + (size_t)slotA * 32 + 16);
        }
        if (activeB) {
          kB = ld_b128_cached(memo.table + (size_t)slotB * 32);
          valB = ld_b128_cached(memo.table + (size_t)slotB * 32 + 16);
        }
        if (activeA) hitA = exp_probe_finish<SMALL>(memo, keyA, slotA, kA, valA);
        if (activeB) hitB = exp_probe_finish<SMALL>(memo, keyB, slotB, kB, valB);
      }
      // --- misses: the merge of a drain round, from the bytes in registers, one word after the other
      bool hardA = false, hardB = false;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        if (!(h ? activeB && !hitB : activeA && !hitA)) continue;
        const U128 key = h ? keyB : keyA;
        const unsigned long long lo = (key.lo >> 8) | (key.hi << 56), hi = key.hi >> 8;
        const int n = (int)(key.lo & 0x7Fu);
        int m = 0;
        if (key.lo & 0x80u) { sm.S[lane] = T.space_sym; m = 1; }
        for (int i = 0; i < n; ++i) {
          const uint32_t c = (uint32_t)((i < 8 ? lo >> (8 * i) : hi >> (8 * (i - 8))) & 0xFFull);
          sm.S[(m++) * 32 + lane] = __ldg(T.ascii_sym + c);
        }
        const uint32_t alive = lane_merge<SMALL>(T, sm, m, lane);
        const int k = __popc(alive);
        uint32_t id[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        bool hard = k > MemoIds<SMALL>::kMax;
        int q = 0;
        for (uint32_t mm = alive; mm && !hard; ++q) {
          const int j = __ffs(mm) - 1;
          mm &= mm - 1;
          const uint32_t sym = sm.S[j * 32 + lane];
          int32_t e = -1;
          if (!(sym & kSymUnknownFlag)) e = __ldg(T.emit + sym);
          if (e < 0 || (uint32_t)e >= (SMALL ? (1u << 16) : (1u << 28))) hard = true;   // unknown / byte fallback: buffer path
          else id[q] = (uint32_t)e;
        }
        if (!hard) {
          const U128 val = MemoIds<SMALL>::pack(k, id);
          if (h) valB = val;
          else valA = val;
          if constexpr (MEMO) {
            uint32_t slot = memo_slot(key, memo.mask);
            const U128 zero{0ull, 0ull};
#pragma unroll 1
            for (int way = 0; way < 2; ++way, slot ^= 1u) {
              uint8_t* e = memo.table + (size_t)slot * 32;
              const U128 old = cas_b128(e, zero, key);
              if ((old.lo | old.hi) == 0) { st_b128(e + 16, val); break; }   // claimed: publish the ids
              if (old.lo == key.lo && old.hi == key.hi) break;                // another warp owns this word
            }
          }
        }
        if (h) hardB = hard;
        else hardA = hard;
      }
      {
        // a word whose ids do not fit a memo payload: the words in front of it go out now, the word itself through
        // the cooperative path
        const uint32_t hmA = __ballot_sync(kFull, hardA), hmB = __ballot_sync(kFull, hardB);
        EXP_CLOCK(t_probe);
        if (hmA | hmB) {
          const int fh = hmA ? __ffs(hmA) - 1 : 32 + __ffs(hmB) - 1;
          EXP_STAT(8);
          if (fh == 0) {
            if (long_word(ex[0])) continue;
            break;
          }
          take = fh;
          cons = ex[2 * take];
        }
      }
      // the next window's bytes: in flight while this one's ids are stored (issued after the probes, so that its
      // registers are not live across them)
      w_next = load_window(wb + cons);
#ifdef XLLM_EXP_STATS
      { const uint32_t aA = __ballot_sync(kFull, activeA), aB = __ballot_sync(kFull, activeB);
        const uint32_t hA = __ballot_sync(kFull, hitA), hB = __ballot_sync(kFull, hitB);
        if (lane == 0) { atomicAdd(&g_exp_stats[9], (unsigned long long)(__popc(aA) + __popc(aB))); atomicAdd(&g_exp_stats[10], (unsigned long long)(__popc(hA) + __popc(hB))); if ((aA & ~hA) | (aB & ~hB)) atomicAdd(&g_exp_stats[11], 1ull); } }
#endif
      // --- ids, in order (words 0..31, then 32..63): the counts are 3-bit, so three ballots per half give every
      // lane its offsets
      const int cntA = lane < take ? MemoIds<SMALL>::count(valA) : 0;
      const int cntB = lane + 32 < take ? MemoIds<SMALL>::count(valB) : 0;
      const uint32_t a0 = __ballot_sync(kFull, cntA & 1), a1 = __ballot_sync(kFull, cntA & 2), a2 = __ballot_sync(kFull, cntA & 4);
      const uint32_t c0 = __ballot_sync(kFull, cntB & 1), c1 = __ballot_sync(kFull, cntB & 2), c2 = __ballot_sync(kFull, cntB & 4);
      const int totalA = __popc(a0) + 2 * __popc(a1) + 4 * __popc(a2);
      const int totalB = __popc(c0) + 2 * __popc(c1) + 4 * __popc(c2);
      const int oA = n_out + __popc(a0 & lt) + 2 * __popc(a1 & lt) + 4 * __popc(a2 & lt);
      const int oB = n_out + totalA + __popc(c0 & lt) + 2 * __popc(c1 & lt) + 4 * __popc(c2 & lt);
      const bool fits = n_out + totalA + totalB <= cap;
      exp_store<SMALL>(out, valA, cntA, oA, a1 != 0u, a2 != 0u, fits, cap);
      if (c0 | c1 | c2) exp_store<SMALL>(out, valB, cntB, oB, c1 != 0u, c2 != 0u, fits, cap);
      n_out += totalA + totalB;
      U = false;
#ifdef XLLM_EXP_STATS
      { const unsigned long long t = clock64(); cyc_window += t_vote - t_step; cyc_probe += t_probe - t_vote; cyc_emit += t - t_probe; ++n_timed; }
#endif
      if (take == nstart) S2 = !((__shfl_sync(kFull, ns16, (cons - 1u) >> 4) >> ((cons - 1u) & 15u)) & 1u);
      }
    } else {
      w_next = load_window(wb + cons);
    }
    EXP_STAT(1);
    // --- the state a drain would have left: is_prev_space, and the U+2581 a kept space puts in front of the next word
    P = S2 && (take > 0 || P || !S);
    S = S2;
    v = wb + cons;
    if (v >= vlen) break;
    w = w_next;
    __syncwarp();
  }
#ifdef XLLM_EXP_STATS
  if (lane == 0) {
    atomicAdd(&g_exp_stats[kExpStatTimed], n_timed);
    atomicAdd(&g_exp_stats[kExpStatCycWindow], cyc_window);
    atomicAdd(&g_exp_stats[kExpStatCycProbe], cyc_probe);
    atomicAdd(&g_exp_stats[kExpStatCycEmit], cyc_emit);
  }
#endif
  rs.P = P;
  rs.S = S;
  rs.U = U;
  rs.n_out = n_out;
  __syncwarp();
  return v - A;
}

// The express kernel: every request starts here when the model allows it (split_mode 1, remove_extra_whitespaces,
// normalised text).  A request it carries to the end is finished (a pending U+2581 is the trailing space the
// normalizer strips); one it cannot is handed to the buffer-path kernel with its position, id count and
// whitespace state, through legacy_list / resume.  kExpWarps independent warps per block.
constexpr int kExpWarps = 4;
// 6 blocks of 4 warps: 80 registers, 24 warps per SM (64 registers spill heavily in the 64-word step, 96 leave 20 warps)
#ifndef XLLM_EXP_MIN_BLOCKS
#define XLLM_EXP_MIN_BLOCKS 6
#endif
template <bool SMALL>
__global__ void __launch_bounds__(kExpWarps * 32, XLLM_EXP_MIN_BLOCKS) sp_express_kernel(
    const uint8_t* __restrict__ text, const int64_t* __restrict__ offsets, int n_req, int32_t* __restrict__ ids,
    int64_t ids_stride, int32_t* __restrict__ n_ids, int32_t* __restrict__ status, const __grid_constant__ SpDev T,
    unsigned int* __restrict__ task_counter, int32_t* __restrict__ legacy_list, unsigned int* __restrict__ legacy_count,
    ExpResume* __restrict__ resume, uint8_t* memo_table, uint32_t memo_mask) {
  const MemoRef memo{memo_table, memo_mask};
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using SM = ExpSmemT<SMALL>;
  SM& sm = reinterpret_cast<SM*>(smem_raw)[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  unsigned long long warp_t0 = 0;
  if (T.warp_ns) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(warp_t0));
  for (;;) {
    unsigned int r = 0;
    if (lane == 0) r = atomicAdd(task_counter, 1u);
    r = __shfl_sync(kFull, r, 0);
    if (r >= (unsigned)n_req) break;
    ExpReq rq;
    const int64_t beg = offsets[r];
    rq.src = text + beg;
    rq.len = (uint32_t)(offsets[r + 1] - beg);
    rq.out = T.out_start ? ids + T.out_start[r] : ids + (int64_t)r * ids_stride;
    rq.cap = T.out_cap ? (int64_t)T.out_cap[r] : ids_stride;
    rq.n_out = 0;
    rq.P = T.add_dummy_prefix != 0;
    rq.S = true;   // is_prev_space starts true under remove_extra_whitespaces
    rq.U = false;
    bool failed = false;
    uint32_t pos = 0;
    if (rq.len > 0) pos = express_run<SMALL, true>(T, sm, rq, 0u, lane, memo, &failed);
#ifdef XLLM_EXP_STATS
    if (lane == 0) { atomicAdd(&g_exp_stats[12], (unsigned long long)pos); atomicAdd(&g_exp_stats[13], (unsigned long long)rq.len); atomicAdd(&g_exp_stats[14], failed ? 1ull : 0ull); }
#endif
    if (lane == 0) {
      if (!failed) {
        n_ids[r] = (int32_t)rq.n_out;
        status[r] = rq.n_out > rq.cap ? kEncTruncated : kEncOk;
      } else {
        ExpResume rr;
        rr.pos = pos;
        rr.flags = (rq.P ? 1u : 0u) | (rq.S ? 2u : 0u) | (rq.U ? 4u : 0u);
        rr.n_out = rq.n_out;
        resume[r] = rr;
        legacy_list[atomicAdd(legacy_count, 1u)] = (int32_t)r;
      }
    }
    __syncwarp();
  }
  if (T.warp_ns && lane == 0) {
    unsigned long long t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    T.warp_ns[blockIdx.x * kExpWarps + (threadIdx.x >> 5)] = t1 - warp_t0;
  }
}

// Writes the symbols of the chars of nbuf[ws, we) flat to S[0..n) and returns n.  *overflow (the same in every lane):
// the word has more than kCoopMaxSym chars, and S holds only the first of them.
template <typename SM>
__device__ __forceinline__ int gather_chars(const SpDev& T, SM& sm, int ws, int we, bool* overflow, int lane) {
  const uint8_t* nb = sm.nbuf;
  int n = 0;
  bool over = false;
  for (int base = ws; base < we; base += 32) {
    const int p = base + lane;
    const bool lead = p < we && (T.byte_mode || (nb[p] & 0xC0) != 0x80);
    const uint32_t m = __ballot_sync(kFull, lead);
    const int idx = n + __popc(m & ((1u << lane) - 1));
    if (lead) {
      if (idx < kCoopMaxSym) { uint32_t adv; sm.S[idx] = char_sym(T, nb + p, &adv); }
      else over = true;
    }
    n += __popc(m);
  }
  *overflow = __any_sync(kFull, over);
  __syncwarp();
  return n;
}

// Tokenises the complete words held in nbuf (all words when final) and keeps the incomplete tail.
// HF: word boundaries come from the regex pre-tokenizer (hf_pretok.cuh); returns true when the word list
// filled up and the kept tail has to be scanned again.
// MODE: 0 SentencePiece BPE / tiktoken, 1 HF byte-level BPE (regex pre-tokenizer), 2 SentencePiece Unigram
// WARM: with the warm-up pre-passes (1b below) for natural text.  A template parameter because carrying their state
// through the in-order rounds slows the plain kernel on the headline workload: the launcher picks the WARM kernels
// only when asked to (XLLM_SP_WARM=1).
template <bool SMALL, bool LONG, int MODE, bool MEMO, bool WARM, typename SM>
__device__ bool drain_pass(const SpDev& T, SM& sm, ReqState& rs, bool final, int lane, MemoRef memo) {
  static_assert(!WARM || (MEMO && !LONG && MODE != 2), "the warm-up pre-passes need the memo and the lane path");
  constexpr bool HF = MODE == 1;
  constexpr bool UNI = MODE == 2;
  const uint8_t* nb = sm.nbuf;
  int nlen = rs.nlen;
  if (final && T.remove_extra_ws) {
    // normalizer.cc: "Ignores trailing space" — strip trailing U+2581 from the stream
    while (nlen >= 3 && nb[nlen - 3] == 0xE2 && nb[nlen - 2] == 0x96 && nb[nlen - 1] == 0x81) nlen -= 3;
    if (nlen == 0) { rs.n_out -= rs.trailing_bare; rs.trailing_bare = 0; }
  }
  if (nlen == 0) { rs.nlen = 0; return false; }

  // 1. word starts: recorded by the fast path, or re-derived after any general-path window
  int nwords = 0;
  int hf_tail = 0;
  bool hf_capped = false;
  if constexpr (HF) {
    const HfScan sc = hf_scan(T, sm, nlen, final, lane);
    if (sc.bad) { rs.bad_input = (int8_t)sc.bad; return false; }
    nwords = sc.nwords;
    hf_tail = sc.tail_start;
    hf_capped = sc.capped;
  } else if (!rs.rescan && !(final && nlen != rs.nlen)) {
    nwords = rs.nw;
  } else if (!rs.rescan) {
    // trailing U+2581 were stripped: drop the starts that now lie at or past the end
    nwords = rs.nw;
    while (nwords > 1 && sm.wstart[nwords - 1] >= nlen) --nwords;
  } else {
    for (int base = 0; base < nlen; base += 32) {
      const int p = base + lane;
      bool st = false;
      if (p < nlen) {
        if (p == 0) st = true;
        else if (T.split_mode != 0 && is_space_at(nb, p, nlen)) {
          st = T.split_mode == 1 || !(p >= 3 && is_space_at(nb, p - 3, nlen));
        }
      }
      const uint32_t m = __ballot_sync(kFull, st);
      if (st) sm.wstart[nwords + __popc(m & ((1u << lane) - 1))] = (uint16_t)p;
      nwords += __popc(m);
    }
  }
  __syncwarp();
  if constexpr (!HF) {
    if (lane == 0) sm.wstart[nwords] = (uint16_t)nlen;
    __syncwarp();
  }
  const int complete = HF ? nwords : (final ? nwords : nwords - 1);

  // byte range, symbol count and kind of word w (w < complete)
  auto word_of = [&](int w, int& ws, int& we, int& nsym, bool& special) {
    ws = we = nsym = 0;
    special = false;
    if constexpr (HF) {
      const uint16_t e = sm.wstart[w];
      ws = e & kHfPosMask;
      we = sm.wstart[w + 1] & kHfPosMask;
      special = (e & kHfSpecialWord) != 0;  // the word is an added token
      nsym = special ? 1 : we - ws;         // every byte is a symbol
    } else {
      ws = sm.wstart[w];
      we = sm.wstart[w + 1];
      if (rs.ascii) nsym = (we - ws) - (nb[ws] == 0xE2 ? 2 : 0);  // ASCII + one leading U+2581
      else
        for (int p = ws; p < we; ++p) nsym += T.byte_mode || (nb[p] & 0xC0) != 0x80;
    }
  };
  // The merge path of one word per lane (not an added token): symbols -> lane_merge -> resolve single-id symbols in
  // place -> (MEMO) insert.  Used by the rounds below for memo misses and by the warm-up pre-pass.  Outputs: alive set
  // in the lane's S column, id count, unknown-symbol flags for the cross-word rule, bare-U+2581 flag.
  auto merge_word = [&](int ws, int we, uint32_t& alive, int& cnt, bool& first_unk, bool& last_unk, bool& bare) {
    alive = 0;
    cnt = 0;
    first_unk = last_unk = bare = false;
    bool direct = false;
    if constexpr (HF) {
      if (T.ignore_merges) {  // models/bpe/model.rs: a pre-token that is a vocabulary entry is that token
        const int32_t id = hf_vocab_lookup(T, nb + ws, we - ws);
        if (id >= 0) {
          sm.S[lane] = kResolvedFlag | (uint32_t)id;
          alive = 1u;
          cnt = 1;
          direct = true;
        }
      }
    }
    bool pu = false, first = true;
    if (!direct) {
      int n = 0;
      for (int p = ws; p < we;) {
        uint32_t adv;
        sm.S[n * 32 + lane] = char_sym(T, nb + p, &adv);
        p += adv;
        ++n;
      }
      bare = (we - ws == 3) && n == 1 && sm.S[lane] == T.space_sym;
      alive = lane_merge<SMALL>(T, sm, n, lane);
    }
    // pass 1: resolve every final symbol; single-id symbols are replaced in place by their token id
    // (tagged), so pass 2 only re-derives the rare multi-id (byte fallback) ones
    for (uint32_t m = direct ? 0u : alive; m;) {
      const int j = __ffs(m) - 1;
      m &= m - 1;
      int32_t tmp[4];
      bool unk;
      const uint32_t sym = sm.S[j * 32 + lane];
      const int c = sym_ids(T, sym, tmp, &unk);
      if (first) { first_unk = unk; first = false; }
      if (!unk && c == 1) sm.S[j * 32 + lane] = kResolvedFlag | (uint32_t)tmp[0];
      if (!(unk && pu && !T.byte_fallback)) cnt += c;
      pu = unk;
    }
    last_unk = pu;
    if constexpr (MEMO) {
      // memoise: every surviving symbol resolved to exactly one id, at most kMax of them
      const int k = __popc(alive);
      U128 key;
      if (k >= 1 && k <= MemoIds<SMALL>::kMax && k == cnt && !bare && memo_key(nb, ws, we, T.byte_mode, &key)) {
        uint32_t id[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        bool ok = true;
        int q = 0;
        for (uint32_t m = alive; m; ++q) {
          const int j = __ffs(m) - 1;
          m &= m - 1;
          const uint32_t sym = sm.S[j * 32 + lane];
          ok = ok && (sym & 0xC0000000u) == kResolvedFlag && (sym & 0x3FFFFFFFu) < (SMALL ? (1u << 16) : (1u << 28));
          id[q] = sym & 0x0FFFFFFFu;
        }
        if (ok) {
          const U128 val = MemoIds<SMALL>::pack(k, id);
          uint32_t slot = memo_slot(key, memo.mask);
          const U128 zero{0ull, 0ull};
#pragma unroll 1
          for (int way = 0; way < 2; ++way, slot ^= 1u) {
            uint8_t* e = memo.table + (size_t)slot * 32;
            const U128 old = cas_b128(e, zero, key);
            if ((old.lo | old.hi) == 0) { st_b128(e + 16, val); break; }   // claimed: publish the ids
            if (old.lo == key.lo && old.hi == key.hi) break;                // another warp owns this word
          }
        }
      }
    }
  };

  // 1b. warm-up pre-passes (throughput kernel with a memo; natural text).  The rounds below go through the words in
  // order, 32 at a time, and a round runs at the speed of its slowest lane: ONE memo miss costs the whole round a merge,
  // and a word beyond the lane columns cuts the round short and is merged by the whole warp on its own.  On the
  // synthetic headline text both are rare; on real text 91 % of the rounds hold a miss and every tenth word is long.
  // So, when the previous drain looked like that:
  //   A1  probe the memo for every short word of the drain first, collect the misses and merge them 32 at a time in FULL
  //       rounds (results go to the memo only); the in-order rounds then find them there;
  //   A2  merge every long word (17..512 symbols) ahead of the rounds and park its ids in a per-warp global scratch
  //       (slot = the word's byte offset: ids never outnumber bytes); in the rounds such a word is an ordinary lane
  //       whose ids are read back from there, so the rounds are no longer cut.  Only for vocabularies without
  //       cross-word unknown merging (byte fallback, or byte-level), where a word's ids do not depend on its neighbours.
  int32_t* arena = nullptr;
  uint16_t* lcnt = nullptr;
  int a1_misses = 0;
  if constexpr (WARM) {
    if (T.warm_arena != nullptr && (rs.warm || rs.had_long)) {
      uint8_t* slice = T.warm_arena + (size_t)blockIdx.x * kWarmSliceBytes;
      const bool do_long = rs.had_long && (T.byte_fallback || T.byte_mode);
      if (do_long) {
        arena = reinterpret_cast<int32_t*>(slice);
        lcnt = reinterpret_cast<uint16_t*>(slice + (size_t)kNBuf * 4);
      }
      int np = 0;  // words waiting in sm.pend[0 .. np)
      auto flush = [&]() {
        __syncwarp();
        int ws = 0, we = 0, nsym = 0;
        bool special = false;
        if (lane < np) word_of(sm.pend[lane], ws, we, nsym, special);
        uint32_t alive;
        int cnt;
        bool fu, lu, bare;
        if (lane < np) merge_word(ws, we, alive, cnt, fu, lu, bare);   // A1 never holds an added token
        np = 0;
        __syncwarp();
      };
      for (int base = 0; base < complete; base += 32) {
        const int w = base + lane;
        const bool have = w < complete;
        int ws = 0, we = 0, nsym = 0;
        bool special = false;
        if (have) word_of(w, ws, we, nsym, special);
        const bool is_long = have && !special && nsym > SM::kRows;
        // ---- A2: the long words of this block, one at a time, whole warp
        uint32_t lm = __ballot_sync(kFull, do_long && is_long);
        while (lm) {
          const int b = __ffs(lm) - 1;
          lm &= lm - 1;
          const int lws = __shfl_sync(kFull, ws, b), lwe = __shfl_sync(kFull, we, b);
          bool overflow;
          int n = gather_chars(T, sm, lws, lwe, &overflow, lane);
          int total = -1;   // ids written for this word, -1: left to the in-order cooperative path
          if (!overflow) {
            int32_t whole = -1;
            if constexpr (HF) {
              if (T.ignore_merges) {
                if (lane == 0) whole = hf_vocab_lookup(T, nb + lws, lwe - lws);
                whole = __shfl_sync(kFull, whole, 0);
              }
            }
            if (whole >= 0) {
              if (lane == 0) arena[lws] = whole;
              total = 1;
            } else {
              n = coop_merge<SMALL>(T, sm, n, lane);
              total = 0;
              for (int sb = 0; sb < n; sb += 32) {
                const int j = sb + lane;
                int32_t tmp[4];
                bool unk = false;
                int c = 0;
                if (j < n) c = sym_ids(T, sm.S[j], tmp, &unk);   // byte fallback: an unknown char is its byte ids
                const int inc2 = warp_incl_scan(c, lane);
                int o = lws + total + (inc2 - c);
                for (int k = 0; k < c; ++k) arena[o++] = tmp[k];
                total += __shfl_sync(kFull, inc2, 31);
              }
            }
          }
          if (lane == 0) lcnt[base + b] = total < 0 ? kNotPre : (uint16_t)total;
          __syncwarp();
        }
        // ---- A1: short words that are not in the memo yet
        if (rs.warm) {
          bool miss = false;
          U128 key;
          if (have && !special && !is_long && memo_key(nb, ws, we, T.byte_mode, &key)) {
            uint32_t slot = memo_slot(key, memo.mask);
            miss = true;
#pragma unroll 1
            for (int way = 0; way < 2; ++way, slot ^= 1u) {
              const U128 k = ld_b128(memo.table + (size_t)slot * 32);
              if (k.lo == key.lo && k.hi == key.hi) { miss = false; break; }
              if ((k.lo | k.hi) == 0) break;
            }
          }
          const uint32_t mm = __ballot_sync(kFull, miss);
          const int k = __popc(mm);
          a1_misses += k;
          if (np + k > 32) flush();
          if (miss) sm.pend[np + __popc(mm & ((1u << lane) - 1))] = (uint16_t)w;
          np += k;
          if (np == 32) flush();
        }
      }
      if (np) flush();
      __syncwarp();
    }
  }

  // 2. rounds of up to 32 consecutive words
  int w0 = 0;
  int n_slow = 0;
  bool long_seen = false;
  while (w0 < complete && !rs.deferred) {
    const int w = w0 + lane;
    const bool have = w < complete;
    int ws = 0, we = 0, nsym = 0;
    bool special = false;  // HF: the word is an added token
    if (have) word_of(w, ws, we, nsym, special);
    // a long word the pre-pass resolved: its ids wait in the arena, it takes part in the round like any other lane
    bool pre = false;
    if constexpr (WARM) pre = arena != nullptr && have && !special && nsym > SM::kRows && lcnt[w] != kNotPre;
    const uint32_t long_mask = __ballot_sync(kFull, have && (UNI || (nsym > SM::kRows && !pre)));  // Unigram: one word at a time
    if constexpr (WARM) long_seen |= long_mask != 0 || __any_sync(kFull, pre);
    const int first_long = long_mask ? __ffs(long_mask) - 1 : 32;
    const bool active = have && lane < first_long;

    // --- fast path: one word per lane
    uint32_t alive = 0;
    int cnt = 0;
    bool first_unk = false, last_unk = false, bare = false;
    bool memo_hit = false;
    if constexpr (MEMO) {
      U128 key;
      if (active && !special && !pre && memo_key(nb, ws, we, T.byte_mode, &key)) {
        uint32_t slot = memo_slot(key, memo.mask);
#pragma unroll 1
        for (int way = 0; way < 2; ++way, slot ^= 1u) {
          const uint8_t* e = memo.table + (size_t)slot * 32;
          const U128 k = ld_b128(e);
          const U128 v = ld_b128(e + 16);
          if (k.lo == key.lo && k.hi == key.hi) {
            if (MemoIds<SMALL>::valid(v)) {
              memo_hit = true;
              cnt = MemoIds<SMALL>::count(v);
              alive = (1u << cnt) - 1u;
#pragma unroll
              for (int q = 0; q < MemoIds<SMALL>::kMax; ++q)
                if (q < cnt) sm.S[q * 32 + lane] = kResolvedFlag | MemoIds<SMALL>::id(v, q);
            }
            break;
          }
          if ((k.lo | k.hi) == 0) break;  // empty: the word was not seen yet
        }
      }
    }
#ifdef XLLM_MEMO_STATS
    {
      const uint32_t am = __ballot_sync(kFull, active), hm = __ballot_sync(kFull, memo_hit);
      if (lane == 0) {
        atomicAdd(&g_memo_stats[0], 1ull);                       // rounds
        atomicAdd(&g_memo_stats[1], (unsigned long long)__popc(am));   // active words
        atomicAdd(&g_memo_stats[2], (unsigned long long)__popc(hm));   // hits
        if (am & ~hm) atomicAdd(&g_memo_stats[3], 1ull);         // rounds with a slow-path lane
        if (first_long < 32) atomicAdd(&g_memo_stats[4], 1ull);  // rounds cut by a long word
      }
    }
#endif
    if (pre && active) {
      cnt = lcnt[w];   // ids parked in the arena by the pre-pass (byte fallback / byte level: no unknown merging)
    } else if (memo_hit) {
    } else if (HF && active && special) {
      int32_t id = 0;
      hf_added_len(T, nb + ws, we - ws, &id);
      sm.S[lane] = kResolvedFlag | (uint32_t)id;
      alive = 1u;
      cnt = 1;
    } else if (active) {
      merge_word(ws, we, alive, cnt, first_unk, last_unk, bare);
    }
    if constexpr (WARM) {
      if (__any_sync(kFull, active && !pre && !memo_hit && !special)) ++n_slow;
    }
    // cross-word unknown merging (byte_fallback off): drop the first id if the previous symbol was unknown too
    bool drop_first = false;
    if (!T.byte_fallback) {
      const uint32_t act_mask = __ballot_sync(kFull, active);
      const uint32_t lu_mask = __ballot_sync(kFull, active && last_unk);
      if (active && first_unk) {
        const bool prev = lane == 0 ? rs.prev_unk : ((lu_mask >> (lane - 1)) & 1u);
        if (prev) { drop_first = true; cnt -= 1; }
      }
      if (act_mask) rs.prev_unk = (lu_mask >> (31 - __clz(act_mask))) & 1u;
    }
    const int incl = warp_incl_scan(cnt, lane);
    const int total = __shfl_sync(kFull, incl, 31);
    if (active && pre) {
      int64_t o = rs.n_out + (incl - cnt);
      for (int q = 0; q < cnt; ++q) put_id(rs, o++, arena[ws + q]);
    } else if (active) {
      int64_t o = rs.n_out + (incl - cnt);
      bool pu = false, first = true;
      for (uint32_t m = alive; m;) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        const uint32_t sym = sm.S[j * 32 + lane];
        if ((sym & 0xC0000000u) == kResolvedFlag) {  // known symbol: one id
          put_id(rs, o++, (int32_t)(sym & 0x3FFFFFFFu));
          pu = false;
        } else {
          int32_t tmp[4];
          bool unk;
          const int c = sym_ids(T, sym, tmp, &unk);
          const bool skip = (unk && pu && !T.byte_fallback) || (first && drop_first);
          if (!skip)
            for (int k = 0; k < c; ++k) put_id(rs, o++, tmp[k]);
          pu = unk;
        }
        first = false;
      }
    }
    rs.n_out += total;
    // trailing bare-word bookkeeping: ids of the run of bare words at the end of what was emitted
    {
      const uint32_t act_mask = __ballot_sync(kFull, active);
      const uint32_t nonbare = __ballot_sync(kFull, active && !bare);
      if (act_mask) {
        const int last_nb = nonbare ? 31 - __clz(nonbare) : -1;  // last non-bare lane
        const int tail = __shfl_sync(kFull, incl, 31) - (last_nb >= 0 ? __shfl_sync(kFull, incl, last_nb) : 0);
        rs.trailing_bare = (last_nb >= 0 ? 0 : rs.trailing_bare) + tail;
      }
    }
    __syncwarp();
    w0 += first_long < 32 ? first_long : 32;
    if (w0 >= complete || first_long == 32) continue;

    // --- cooperative path for the long word w0
    {
      const int lws = HF ? (sm.wstart[w0] & kHfPosMask) : sm.wstart[w0];
      int lwe = HF ? (sm.wstart[w0 + 1] & kHfPosMask) : sm.wstart[w0 + 1];
      int words_taken = 1;
      if constexpr (UNI) {
        auto is_bare = [&](int a, int b) { return b - a == 3 && nb[a] == 0xE2 && nb[a + 1] == 0x96 && nb[a + 2] == 0x81; };
        const bool bare_word = is_bare(lws, lwe);
        // No piece spans a word start, so consecutive words form one lattice: take as many complete words as the
        // lattice scratch holds — the trie walks then fill all 32 lanes and the per-word overhead is paid once per run.
        // A bare U+2581 word stays on its own (trailing-space bookkeeping).
        if (!bare_word) {
          while (w0 + words_taken < complete) {
            const int a = sm.wstart[w0 + words_taken], b = sm.wstart[w0 + words_taken + 1];
            if (b - lws > kUniMaxWord || is_bare(a, b)) break;
            lwe = b;
            ++words_taken;
          }
        }
        const int len = lwe - lws;
        if (len > kUniMaxWord) {
          rs.too_long = true;  // the Viterbi lattice of one word lives in shared memory
        } else {
          const int n = unigram_word(T, sm, nb + lws, len, &rs.uni_score, lane);
          const int64_t before = rs.n_out;
          for (int base = 0; base < n; base += 32) {
            const int j = base + lane;
            int32_t tmp[4];
            bool unk = false;
            int c = 0;
            if (j < n) {
              const uint32_t sym = sm.S[j];
              if ((sym & 0xC0000000u) == kResolvedFlag) { tmp[0] = (int32_t)(sym & 0x3FFFFFFFu); c = 1; }
              else c = sym_ids(T, sym, tmp, &unk);
            }
            bool skip = false;
            if (!T.byte_fallback) {
              const uint32_t um = __ballot_sync(kFull, j < n && unk);
              const bool prev = lane == 0 ? rs.prev_unk : ((um >> (lane - 1)) & 1u);
              skip = unk && prev;
              const int lastl = (n - base) >= 32 ? 31 : (n - base - 1);
              rs.prev_unk = (um >> lastl) & 1u;
            }
            if (skip) c = 0;
            const int inc2 = warp_incl_scan(c, lane);
            int64_t o = rs.n_out + (inc2 - c);
            for (int k = 0; k < c; ++k) put_id(rs, o++, tmp[k]);
            rs.n_out += __shfl_sync(kFull, inc2, 31);
          }
          rs.trailing_bare = bare_word ? rs.trailing_bare + (int32_t)(rs.n_out - before) : 0;
        }
      } else {
        bool overflow;
        int n = gather_chars(T, sm, lws, lwe, &overflow, lane);
        int32_t whole = -1;
        if constexpr (HF) {
          if (T.ignore_merges && !overflow) {  // no vocabulary entry is longer than the cooperative path (host check)
            if (lane == 0) whole = hf_vocab_lookup(T, nb + lws, lwe - lws);
            whole = __shfl_sync(kFull, whole, 0);
          }
        }
        if (whole >= 0) {
          if (lane == 0) put_id(rs, rs.n_out, whole);
          rs.n_out += 1;
          rs.trailing_bare = 0;
        } else if (overflow) {
          // more chars than the shared-memory scratch holds: merge it in a global scratch slot
          if constexpr (!LONG) {
            rs.deferred = true;
          } else if (T.long_slots <= 0) {
            rs.too_long = true;
          } else {
            rs.long_slot = long_slot_acquire(T.long_locks, T.long_slots, lane);
            rs.long_n = 0;
            if (long_append(T, sm, rs, lws, lwe, lane)) long_finish(T, rs, false, lane);
            else rs.too_long = true;
            long_slot_release(T.long_locks, rs.long_slot, lane);
          }
        } else {
          n = coop_merge<SMALL>(T, sm, n, lane);
          for (int base = 0; base < n; base += 32) {
            const int j = base + lane;
            int32_t tmp[4];
            bool unk = false;
            int c = 0;
            if (j < n) c = sym_ids(T, sm.S[j], tmp, &unk);
            bool skip = false;
            if (!T.byte_fallback) {
              const uint32_t um = __ballot_sync(kFull, j < n && unk);
              const bool prev = lane == 0 ? rs.prev_unk : ((um >> (lane - 1)) & 1u);
              skip = unk && prev;
              const int lastl = (n - base) >= 32 ? 31 : (n - base - 1);
              rs.prev_unk = (um >> lastl) & 1u;
            }
            if (skip) c = 0;
            const int inc2 = warp_incl_scan(c, lane);
            int64_t o = rs.n_out + (inc2 - c);
            for (int k = 0; k < c; ++k) put_id(rs, o++, tmp[k]);
            rs.n_out += __shfl_sync(kFull, inc2, 31);
          }
          rs.trailing_bare = 0;
        }
      }
      __syncwarp();
      w0 += words_taken;
    }
  }

  // 3. keep the incomplete tail at the front of nbuf
  if (!final || (HF && hf_tail < nlen)) {
    const int ts = HF ? hf_tail : sm.wstart[nwords - 1];
    const int tl = nlen - ts;
    if (ts > 0) {
      for (int base = 0; base < tl; base += 32) {
        const int k = base + lane;
        uint8_t c = 0;
        if (k < tl) c = sm.nbuf[ts + k];
        __syncwarp();
        if (k < tl) sm.nbuf[k] = c;
        __syncwarp();
      }
    }
    rs.nlen = tl;
    __syncwarp();  // every lane has read wstart[nwords - 1] (which is wstart[0] when one word is left)
    if (lane == 0) sm.wstart[0] = 0;
    rs.nw = 1;
    if (!rs.ascii) {  // the kept tail decides whether the buffer is ASCII-only again
      bool non_ascii = false;
      const bool lead = tl >= 3 && sm.nbuf[0] == 0xE2 && sm.nbuf[1] == 0x96 && sm.nbuf[2] == 0x81;
      for (int k = lane; k < tl; k += 32) non_ascii |= sm.nbuf[k] >= 0x80 && !(lead && k < 3);
      rs.ascii = !T.byte_mode && !__any_sync(kFull, non_ascii);
    }
  } else {
    rs.nlen = 0;
    rs.nw = 0;
    rs.ascii = !T.byte_mode;
  }
  rs.rescan = false;
  if constexpr (WARM) {
    // the next drain of this request (and, carried over, the next request of the batch) warms up when this one paid
    // for misses, and resolves long words ahead when this one had any
    rs.warm = n_slow >= 2 || a1_misses >= 8;
    rs.had_long = long_seen;
  }
  __syncwarp();
  return HF && hf_capped && !rs.deferred;
}

template <bool SMALL, bool LONG, int MODE, bool MEMO, bool WARM, typename SM>
__device__ __forceinline__ void drain(const SpDev& T, SM& sm, ReqState& rs, bool final, int lane, MemoRef memo) {
  if constexpr (MODE == 1) {
    while (drain_pass<SMALL, LONG, 1, MEMO, WARM>(T, sm, rs, final, lane, memo)) {}
  } else {
    drain_pass<SMALL, LONG, MODE, MEMO, WARM>(T, sm, rs, final, lane, memo);
  }
}

// LONG == false: the throughput kernel; a request that needs the long-word path is appended to defer_list.
// LONG == true : re-runs exactly the deferred requests (work list = defer_list[0 .. *defer_count)).
// HF == true : byte-level BPE with the regex pre-tokenizer (split_mode 3).
// MEMO == true: words are looked up in / added to the launch's word memo (never built together with LONG).
// WARM == true: drains run the warm-up pre-passes of drain_pass (natural text; MEMO kernels only).
template <bool SMALL, bool LONG, int MODE, bool MEMO, bool WARM = false>
__global__ void __launch_bounds__(32, LONG ? 8 : ((MODE != 2 && !WARM) ? 16 : 27)) sp_encode_kernel(
    const uint8_t* __restrict__ text, const int64_t* __restrict__ offsets, int n_req, int32_t* __restrict__ ids,
    int64_t ids_stride, int32_t* __restrict__ n_ids, int32_t* __restrict__ status, const __grid_constant__ SpDev T,
    unsigned int* __restrict__ task_counter, int32_t* __restrict__ defer_list,
    unsigned int* __restrict__ defer_count, uint8_t* memo_table, uint32_t memo_mask) {
  constexpr bool HF = MODE == 1;
  const MemoRef memo{memo_table, memo_mask};
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using SM = typename std::conditional<MODE == 2, WarpSmemUniT<SMALL>, WarpSmemT<SMALL, (MODE != 2 && !WARM) ? kHfRows : kMaxSym>>::type;
  SM& sm = *reinterpret_cast<SM*>(smem_raw);
  const int lane = threadIdx.x;
  const int drain_at = kNBuf - 3 * kFastWin - 8;  // room for one more fast-path step
  bool warm_carry = false, long_carry = false;   // WARM: what the previous request's text looked like (same batch)
  unsigned long long warp_t0 = 0;
  if constexpr (!LONG) {
    if (T.warp_ns) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(warp_t0));
  }

  for (;;) {
    unsigned int r = 0;
    if (lane == 0) r = atomicAdd(task_counter, 1u);
    r = __shfl_sync(kFull, r, 0);
    if constexpr (LONG) {
      if (r >= *defer_count) break;
      r = (unsigned)defer_list[r];
    } else if (T.work_list) {   // the requests the express kernel handed over
      if (r >= *T.work_count) break;
      r = (unsigned)T.work_list[r];
    } else {
      if (r >= (unsigned)n_req) break;
    }

    ReqState rs;
    const int64_t beg = offsets[r];
    rs.src = text + beg;
    rs.len = (uint32_t)(offsets[r + 1] - beg);
    rs.out = T.out_start ? ids + T.out_start[r] : ids + (int64_t)r * ids_stride;
    rs.cap = T.out_cap ? (int64_t)T.out_cap[r] : ids_stride;
    rs.n_out = 0;
    rs.nlen = 0;
    rs.trailing_bare = 0;
    rs.nw = 0;
    rs.rescan = false;
    rs.ascii = !T.byte_mode;
    rs.prev_space = T.remove_extra_ws;
    rs.prev_unk = false;
    rs.too_long = false;
    rs.bad_input = 0;
    rs.uni_score = 0.f;
    rs.deferred = false;
    rs.warm = warm_carry;
    rs.had_long = long_carry;
    rs.long_mode = false;
    rs.long_last_sp = false;
    rs.long_slot = -1;
    rs.long_n = 0;

    if constexpr (HF) {
      // TemplateProcessing ids in front (add_special_tokens = 1, fast_tokenizer.cpp:24), also for an empty text
      if (lane < T.n_prefix) put_id(rs, lane, T.prefix_ids[lane]);
      rs.n_out = T.n_prefix;
      if (lane == 0) sm.wstart[0] = 0;
      for (uint32_t pos = 0; pos < rs.len; pos += kFastWin) {
        normalize_fast(T, sm, rs, pos, lane);  // byte mode: a verbatim copy
        if (rs.nlen > drain_at) {
          drain<SMALL, LONG, 1, MEMO, WARM>(T, sm, rs, false, lane, memo);
          // what is left is one unfinished pre-token (plus the look-ahead margin)
          if (rs.nlen > kLongEnterAt) rs.too_long = true;
          if (rs.too_long || rs.deferred || rs.bad_input) break;
        }
      }
      if (!rs.too_long && !rs.deferred && !rs.bad_input) drain<SMALL, LONG, 1, MEMO, WARM>(T, sm, rs, true, lane, memo);
      if (!rs.too_long && !rs.deferred && !rs.bad_input) {
        if (lane < T.n_suffix) put_id(rs, rs.n_out + lane, T.suffix_ids[lane]);
        rs.n_out += T.n_suffix;
      }
    } else if (rs.len > 0) {
      bool lead_space = T.add_dummy_prefix;
      uint32_t pos0 = 0;
      if constexpr (MODE == 0) {
        if (T.resume) {   // taken over from the express kernel: its ids are in the row, a pending U+2581 leads the next word
          const ExpResume rr = reinterpret_cast<const ExpResume*>(T.resume)[r];
          pos0 = rr.pos;
          rs.n_out = rr.n_out;
          lead_space = (rr.flags & 1u) != 0;
          rs.prev_space = (rr.flags & 2u) != 0;
          rs.prev_unk = (rr.flags & 4u) != 0;
        }
      }
      if (lead_space) {
        if (lane == 0) { sm.nbuf[0] = 0xE2; sm.nbuf[1] = 0x96; sm.nbuf[2] = 0x81; sm.wstart[0] = 0; }
        rs.nlen = 3;
        rs.nw = 1;
      }
      __syncwarp();
      uint32_t carry_skip = 0;
      for (uint32_t pos = pos0; pos < rs.len;) {
        if (carry_skip == 0 && normalize_fast(T, sm, rs, pos, lane)) {
          pos += kFastWin;
        } else {
          if (!normalize_window(T, sm, rs, pos, carry_skip, lane)) {
            // make room, then this window must fit
            bool consumed = false;
            if constexpr (LONG) {
              if (rs.long_mode) { long_consume(T, sm, rs, false, lane); consumed = true; }
            }
            if (!consumed) drain<SMALL, LONG, MODE, MEMO, WARM>(T, sm, rs, false, lane, memo);
            if (!rs.too_long && !normalize_window(T, sm, rs, pos, carry_skip, lane)) {
              // still no room: the kept tail is one very long word -> stream it through a scratch slot
              bool entered = false;
              if constexpr (LONG) {
                if (!rs.long_mode) entered = long_enter(T, sm, rs, lane);
                if (!entered) rs.too_long = true;
              } else {
                rs.deferred = true;  // needs the long-word kernel
              }
              if (entered && !normalize_window(T, sm, rs, pos, carry_skip, lane)) rs.too_long = true;
            }
            if (rs.too_long || rs.deferred) break;
          }
          pos += 32;
        }
        bool in_long = false;
        if constexpr (LONG) {
          if (rs.long_mode) {
            in_long = true;
            if (rs.nlen > kLongFlushAt) long_consume(T, sm, rs, false, lane);
          }
        }
        if (!in_long && rs.nlen > drain_at) {
          drain<SMALL, LONG, MODE, MEMO, WARM>(T, sm, rs, false, lane, memo);
          if (rs.nlen > kLongEnterAt) {
            if constexpr (LONG) {
              if (!long_enter(T, sm, rs, lane)) rs.too_long = true;
            } else {
              rs.deferred = true;
            }
          }
        }
        if (rs.too_long || rs.deferred) break;
      }
      if constexpr (LONG) {
        if (!rs.too_long && rs.long_mode) long_consume(T, sm, rs, true, lane);
      }
      if (!rs.too_long && !rs.deferred) drain<SMALL, LONG, MODE, MEMO, WARM>(T, sm, rs, true, lane, memo);
    }
    if constexpr (LONG) {
      if (rs.long_mode) {  // error exit while a slot is held
        long_slot_release(T.long_locks, rs.long_slot, lane);
        rs.long_mode = false;
      }
    }
    if constexpr (MODE == 2) {
      if (rs.deferred) { rs.deferred = false; rs.too_long = true; }  // no long-word pass for Unigram
    }
    warm_carry = rs.warm;
    long_carry = rs.had_long;
    if (lane == 0) {
      if (rs.deferred) {
        defer_list[atomicAdd(defer_count, 1u)] = (int32_t)r;
        n_ids[r] = 0;
        status[r] = kEncWordTooLong;  // overwritten by the long-word kernel
      } else {
        const bool failed = rs.too_long || rs.bad_input;
        n_ids[r] = failed ? 0 : (int32_t)rs.n_out;
        status[r] = rs.bad_input ? (rs.bad_input == 1 ? kEncBadUtf8 : kEncNeedsNfc)
                                 : (rs.too_long ? kEncWordTooLong : (rs.n_out > rs.cap ? kEncTruncated : kEncOk));
      }
    }
    __syncwarp();
  }
  if constexpr (!LONG) {
    if (T.warp_ns && lane == 0) {
      unsigned long long t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      T.warp_ns[blockIdx.x] += t1 - warp_t0;   // on top of the express kernel's share, if it ran (the caller zeroes the array)
    }
  }
}

}  // namespace

// ------------------------------------------------------------------------------ host side
#ifdef XLLM_EXP_STATS
extern "C" void xllm_debug_exp_stats(unsigned long long* out) {
  cudaMemcpyFromSymbol(out, g_exp_stats, sizeof(unsigned long long) * kExpStats);
  unsigned long long z[kExpStats] = {0};
  cudaMemcpyToSymbol(g_exp_stats, z, sizeof(z));
}
#endif
#ifdef XLLM_MEMO_STATS
extern "C" void xllm_debug_memo_stats(unsigned long long* out) {
  cudaMemcpyFromSymbol(out, g_memo_stats, sizeof(unsigned long long) * 8);
  unsigned long long z[8] = {0};
  cudaMemcpyToSymbol(g_memo_stats, z, sizeof(z));
}
#endif
uint32_t sp_memo_default_slots() {
  uint32_t slots = 1u << 18;
  if (const char* w = getenv("XLLM_SP_MEMO_SLOTS")) {
    const long v = atol(w);
    if (v <= 0) return 0;
    slots = 2;
    while (slots < (uint32_t)v && slots < (1u << 26)) slots <<= 1;
  }
  return slots;
}

SpDeviceModel::~SpDeviceModel() {
  for (int i = 0; i < n_allocs_; ++i) cudaFree(allocs_[i]);
}

int SpDeviceModel::upload(const SpTables& t) {
  if (t.split_mode == 3 && (!t.byte_mode || t.added_tokens.size() > 256 || t.uni_stage1.empty())) {
    set_last_error("split_mode 3 (regex pre-tokenizer) needs byte-mode tables and the Unicode class tables");
    return XLLM_ERR_UNSUPPORTED;
  }
  if (32 * t.max_unit_out + 64 > (uint32_t)kNBuf) {
    set_last_error("normalizer replacement of %u bytes exceeds the device staging budget", t.max_unit_out);
    return XLLM_ERR_UNSUPPORTED;
  }
  auto up = [&](const void* src, size_t bytes, const void** dst) -> int {
    void* d = nullptr;
    const size_t alloc = bytes ? bytes : 16;
    cudaError_t e = cudaMalloc(&d, alloc);
    if (e != cudaSuccess) {
      set_last_error("cudaMalloc(%zu) for tokenizer tables failed: %s", alloc, cudaGetErrorString(e));
      return XLLM_ERR_NOMEM;
    }
    allocs_[n_allocs_++] = d;
    if (bytes) {
      e = cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice);
      if (e != cudaSuccess) {
        set_last_error("cudaMemcpy of tokenizer tables failed: %s", cudaGetErrorString(e));
        return XLLM_ERR_CUDA;
      }
    }
    *dst = d;
    return XLLM_OK;
  };
  int rc;
#define UP(vec, field)                                                                                      \
  if ((rc = up((vec).data(), (vec).size() * sizeof((vec)[0]), reinterpret_cast<const void**>(&dev_.field))) != \
      XLLM_OK)                                                                                              \
    return rc;
  UP(t.trie, trie);
  UP(t.blob, blob);
  UP(t.ascii_sym, ascii_sym);
  UP(t.cp_table, cp_table);
  UP(t.pair_table, pair_table);
  UP(t.emit, emit);
  UP(t.virt_cp, virt_cp);
  UP(t.byte_id, byte_id);
  UP(t.uni_stage1, uni1);
  UP(t.uni_stage2, uni2);
  {
    std::vector<uint8_t> blob;
    std::vector<uint16_t> off(1, 0);
    std::vector<int32_t> aid;
    for (const auto& a : t.added_tokens) {
      blob.insert(blob.end(), a.first.begin(), a.first.end());
      off.push_back((uint16_t)blob.size());
      aid.push_back(a.second);
      dev_.added_first[(uint8_t)a.first[0] >> 5] |= 1u << ((uint8_t)a.first[0] & 31);
      if (a.first.size() > dev_.added_max_len) dev_.added_max_len = (uint32_t)a.first.size();
    }
    dev_.n_added = (uint32_t)aid.size();
    UP(blob, added_blob);
    UP(off, added_off);
    UP(aid, added_id);
  }
  dev_.ignore_merges = t.ignore_merges ? 1 : 0;
  dev_.unigram = t.unigram ? 1 : 0;
  if (t.unigram) {
    UP(t.piece_score, piece_score);
    UP(t.uni_trie, utrie);
    dev_.utrie_mask = (uint32_t)(t.uni_trie.size() / 4) - 1;
    dev_.unk_score = t.unk_score;
    dev_.max_piece_len = t.max_piece_len;
  }
  if (t.ignore_merges || t.unigram) {
    UP(t.vocab_table, vtab);
    UP(t.vocab_blob, vblob);
    dev_.vtab_mask = (uint32_t)(t.vocab_table.size() / 4) - 1;
  }
  dev_.nfc_check = t.nfc_check ? 1 : 0;
  dev_.hf_pattern = (uint8_t)t.hf_pattern;
  dev_.hf_digits = (uint8_t)(t.hf_digits > 0 ? t.hf_digits : 1);
  dev_.n_prefix = (uint8_t)t.prefix_ids.size();
  dev_.n_suffix = (uint8_t)t.suffix_ids.size();
  for (size_t i = 0; i < t.prefix_ids.size() && i < 4; ++i) dev_.prefix_ids[i] = t.prefix_ids[i];
  for (size_t i = 0; i < t.suffix_ids.size() && i < 4; ++i) dev_.suffix_ids[i] = t.suffix_ids[i];
#undef UP
  dev_.trie_units = (uint32_t)t.trie.size();
  dev_.cp_mask = (uint32_t)t.cp_table.size() - 1;
  dev_.pair_mask = (uint32_t)t.pair_table.size() - 1;
  {
    uint32_t lg = 0;
    while ((1u << lg) < (uint32_t)t.pair_table.size()) ++lg;
    dev_.pair_shift = 32 - lg;
  }
  dev_.n_pieces = t.n_pieces;
  dev_.space_sym = t.space_sym;
  dev_.unk_id = t.unk_id;
  dev_.max_unit_out = t.max_unit_out;
  uint32_t max_rank = 0;
  for (const auto& e : t.pair_table)
    if (e.a != kEmptyKey && e.prio > max_rank) max_rank = e.prio;
  dev_.small_vocab = (t.n_pieces < 65535 && max_rank < 65535) ? 1 : 0;
  if (const char* w = getenv("XLLM_SP_FORCE_WIDE"))  // tests: run a small vocabulary through the 32-bit-state kernels
    if (atoi(w) != 0) dev_.small_vocab = 0;
  dev_.express = 1;
  if (const char* w = getenv("XLLM_SP_EXPRESS")) dev_.express = atoi(w) != 0 ? 1 : 0;   // 0: every window takes the buffer path
  // scratch pool for pre-tokens longer than the shared-memory paths hold
  uint32_t cap = 1u << 17;
  int slots = 64;
  if (const char* w = getenv("XLLM_SP_LONG_CAP")) cap = (uint32_t)atoi(w);
  if (const char* w = getenv("XLLM_SP_LONG_SLOTS")) slots = atoi(w);
  cap = (cap + 31) & ~31u;
  if (slots > 0 && cap > 0) {
    void* pool = nullptr;
    void* locks = nullptr;
    if (cudaMalloc(&pool, long_slot_bytes(cap) * (size_t)slots) != cudaSuccess ||
        cudaMalloc(&locks, sizeof(int) * (size_t)slots) != cudaSuccess ||
        cudaMemset(locks, 0, sizeof(int) * (size_t)slots) != cudaSuccess) {
      set_last_error("cudaMalloc of the long-word scratch pool (%d x %u symbols) failed", slots, cap);
      if (pool) cudaFree(pool);
      if (locks) cudaFree(locks);
      return XLLM_ERR_NOMEM;
    }
    allocs_[n_allocs_++] = pool;
    allocs_[n_allocs_++] = locks;
    dev_.long_pool = static_cast<uint8_t*>(pool);
    dev_.long_locks = static_cast<int*>(locks);
    dev_.long_cap = cap;
    dev_.long_slots = slots;
  }
  for (int i = 0; i < 4; ++i) dev_.simple_ascii[i] = t.simple_ascii[i];
  for (int i = 0; i < 4; ++i) dev_.spacelike_ascii[i] = t.spacelike_ascii[i];
  dev_.byte_fallback = t.byte_fallback;
  dev_.add_dummy_prefix = t.add_dummy_prefix;
  dev_.remove_extra_ws = t.remove_extra_whitespaces;
  dev_.split_mode = (uint8_t)t.split_mode;
  dev_.byte_mode = t.byte_mode ? 1 : 0;
  {  // printable ASCII (0x20..0x7E) all "simple": the fast path tests a whole word at once
    bool all = true;
    for (uint32_t c = 0x20; c <= 0x7E; ++c) all = all && ((t.simple_ascii[c >> 5] >> (c & 31)) & 1u);
    dev_.printable_simple = all ? 1 : 0;
  }
  return XLLM_OK;
}

// Per device: the SM count, and the resident blocks per SM of the express kernel ([small_vocab]).
static DeviceOnce g_sp_once;
static int g_exp_per_sm[DeviceOnce::kMaxDevices][2];

// Resident one-warp blocks per SM of a buffer-path kernel whose warp takes smem bytes of shared memory: as many as
// 227 KB holds with 1 KB reserved per block, at most 27.
static int sp_warps_per_sm(size_t smem) {
  const int w = (int)((227 * 1024) / (smem + 1024));
  return w > 27 ? 27 : w;
}

// the express kernel runs in front of the buffer-path kernel for these models (and only with the word memo on)
static bool sp_express_model(const SpDev& dev) {
  return dev.express && !dev.unigram && !dev.byte_mode && dev.split_mode == 1 && dev.remove_extra_ws;
}

// One warp's shared memory in sp_encode_kernel<SMALL, ·, MODE, ·, WARM>: the kernel's own SM type.
template <bool SMALL, int MODE, bool WARM>
using EncodeSmem = typename std::conditional<MODE == 2, WarpSmemUniT<SMALL>, WarpSmemT<SMALL, WARM ? kMaxSym : kHfRows>>::type;

template <bool SMALL>
static size_t throughput_smem(bool unigram, bool warm) {
  return unigram ? sizeof(EncodeSmem<SMALL, 2, false>)
                 : (warm ? sizeof(EncodeSmem<SMALL, 0, true>) : sizeof(EncodeSmem<SMALL, 0, false>));
}

cudaError_t sp_encode_plan(const SpDev& dev, int n_req, bool memo, bool warm, SpEncodePlan* plan) {
  SpEncodePlan& p = *plan;
  p = SpEncodePlan();
  cudaError_t e = cudaSuccess;
  int d = 0;   // get() sets it before the setup runs
  const int n_sm = g_sp_once.get(
      [&] {
        for (int s = 0; s < 2; ++s) {
          int& b = g_exp_per_sm[d][s];
          const cudaError_t r =
              s ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, sp_express_kernel<true>, kExpWarps * 32,
                                                                kExpWarps * sizeof(ExpSmemT<true>))
                : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, sp_express_kernel<false>, kExpWarps * 32,
                                                                kExpWarps * sizeof(ExpSmemT<false>));
          if (r != cudaSuccess) return r;
          if (b < 1) b = 1;
        }
        return cudaSuccess;
      },
      &e, &d);
  if (e != cudaSuccess) return e;
  const bool small = dev.small_vocab != 0;
  const int n = n_req > 0 ? n_req : 0;
  // the warm-up pre-passes live in the memo kernels of BPE models; the express kernel has none, so warm replaces it
  p.memo = memo;
  p.warm = warm && memo && !dev.unigram;
  p.express = memo && !p.warm && sp_express_model(dev);
  p.long_pass = !dev.unigram;   // Viterbi has no long-word pass
  p.kernels = 1 + (p.express ? 1 : 0) + (p.long_pass ? 1 : 0);
  const size_t smem = small ? throughput_smem<true>(dev.unigram, p.warm) : throughput_smem<false>(dev.unigram, p.warm);
  const int full_grid = n_sm * sp_warps_per_sm(smem);
  p.grid = full_grid < n ? full_grid : n;
  p.grid_long = n_sm * 2 < n ? n_sm * 2 : n;
  p.warp_ns = p.grid;
  if (p.express) {
    int per_sm = g_exp_per_sm[d][small];
    if (const char* w = getenv("XLLM_SP_EXPRESS_BLOCKS_PER_SM")) {
      const int v = atoi(w);
      if (v > 0 && v < per_sm) per_sm = v;
    }
    const int need = (n + kExpWarps - 1) / kExpWarps;
    p.express_blocks = n_sm * per_sm < need ? n_sm * per_sm : need;
    if (p.express_blocks * kExpWarps > p.warp_ns) p.warp_ns = p.express_blocks * kExpWarps;
  }
  // scratch: [deferred requests n][handed-over requests n, to 16 bytes][resume records n]
  p.scratch_bytes = (((size_t)n * 8 + 15) & ~(size_t)15) + (size_t)n * sizeof(ExpResume) + 16;
  p.arena_bytes = p.warm ? (size_t)full_grid * kWarmSliceBytes : 0;
  return cudaSuccess;
}

// What every kernel of one sp_encode_launch is passed.
struct EncodeArgs {
  const uint8_t* text;
  const int64_t* offsets;
  int n_req;
  int32_t* ids;
  int64_t ids_stride;
  int32_t* n_ids;
  int32_t* status;
  SpDev dev;
  unsigned int* counters;
  void* scratch;
  uint8_t* memo_table;
  uint32_t memo_mask;
  cudaStream_t stream;
};

// Launches sp_encode_kernel<SMALL, LONG, MODE, MEMO, WARM> with one warp per block and that warp's shared memory, the
// size this instantiation is opted in to once per device.
template <bool SMALL, bool LONG, int MODE, bool MEMO, bool WARM>
static cudaError_t launch_encode(int grid, const EncodeArgs& a) {
  constexpr size_t smem = sizeof(EncodeSmem<SMALL, MODE, WARM>);
  static DeviceOnce once;
  cudaError_t e = cudaSuccess;
  once.get(
      [] {
        return cudaFuncSetAttribute(sp_encode_kernel<SMALL, LONG, MODE, MEMO, WARM>,
                                    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      },
      &e);
  if (e != cudaSuccess) return e;
  sp_encode_kernel<SMALL, LONG, MODE, MEMO, WARM><<<grid, 32, smem, a.stream>>>(
      a.text, a.offsets, a.n_req, a.ids, a.ids_stride, a.n_ids, a.status, a.dev, a.counters + (LONG ? 2 : 0),
      static_cast<int32_t*>(a.scratch), a.counters + 1, MEMO ? a.memo_table : nullptr, MEMO ? a.memo_mask : 0u);
  return cudaGetLastError();
}

// BPE: the throughput kernel (memo off, on, or on with the warm-up pre-passes), then the long-word kernel over the
// requests it deferred.
template <bool SMALL, int MODE>
static cudaError_t launch_bpe(const SpEncodePlan& p, const EncodeArgs& a) {
  const cudaError_t e = p.warm   ? launch_encode<SMALL, false, MODE, true, true>(p.grid, a)
                        : p.memo ? launch_encode<SMALL, false, MODE, true, false>(p.grid, a)
                                 : launch_encode<SMALL, false, MODE, false, false>(p.grid, a);
  if (e != cudaSuccess) return e;
  return launch_encode<SMALL, true, MODE, false, false>(p.grid_long, a);
}

// Every kernel the plan lists, in order: the express kernel, whose hand-overs continue in the buffer-path kernels.
template <bool SMALL>
static cudaError_t launch_plan(const SpEncodePlan& p, EncodeArgs a) {
  if (p.express) {
    int32_t* const legacy_list = static_cast<int32_t*>(a.scratch) + a.n_req;
    ExpResume* const resume =
        reinterpret_cast<ExpResume*>(static_cast<uint8_t*>(a.scratch) + (((size_t)a.n_req * 8 + 15) & ~(size_t)15));
    sp_express_kernel<SMALL><<<p.express_blocks, kExpWarps * 32, kExpWarps * sizeof(ExpSmemT<SMALL>), a.stream>>>(
        a.text, a.offsets, a.n_req, a.ids, a.ids_stride, a.n_ids, a.status, a.dev, a.counters + 3, legacy_list,
        a.counters + 4, resume, a.memo_table, a.memo_mask);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    a.dev.work_list = legacy_list;
    a.dev.work_count = a.counters + 4;
    a.dev.resume = resume;
  }
  // Unigram: Viterbi per word from a running score, so no word memo (the result depends on the prefix)
  if (a.dev.unigram) return launch_encode<SMALL, false, 2, false, false>(p.grid, a);
  return a.dev.split_mode == 3 ? launch_bpe<SMALL, 1>(p, a) : launch_bpe<SMALL, 0>(p, a);
}

cudaError_t sp_encode_launch(const SpDev& dev, const uint8_t* text, const int64_t* offsets, int n_req, int32_t* ids,
                             int64_t ids_stride, int32_t* n_ids, int32_t* status, unsigned int* counters,
                             void* scratch, cudaStream_t stream, SpMemo memo, SpLaunchOpts opts) {
  if (n_req <= 0) return cudaSuccess;
  const bool use_memo = memo.table != nullptr && memo.slots >= 2 && (memo.slots & (memo.slots - 1)) == 0;
  SpEncodePlan plan;
  cudaError_t e = sp_encode_plan(dev, n_req, use_memo, memo.warm, &plan);
  if (e != cudaSuccess) return e;
  if (plan.warm && (memo.arena == nullptr || memo.arena_bytes < plan.arena_bytes)) return cudaErrorInvalidValue;
  // the kernels take the table descriptor by value: the per-launch options ride along
  EncodeArgs a{text, offsets, n_req, ids, ids_stride, n_ids, status, dev, counters, scratch,
               plan.memo ? static_cast<uint8_t*>(memo.table) : nullptr, plan.memo ? memo.slots - 1 : 0u, stream};
  a.dev.out_start = opts.out_start;
  a.dev.out_cap = opts.out_cap;
  a.dev.warp_ns = opts.warp_ns;
  a.dev.warm_arena = plan.warm ? static_cast<uint8_t*>(memo.arena) : nullptr;
  a.dev.work_list = nullptr;
  a.dev.work_count = nullptr;
  a.dev.resume = nullptr;
  // counters[0]: task counter, [1]: deferred count, [2]: task counter of the long-word pass,
  // [3]: task counter of the express kernel, [4]: requests it handed over
  e = cudaMemsetAsync(counters, 0, 5 * sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
  if (use_memo && memo.clear) {
    e = cudaMemsetAsync(memo.table, 0, (size_t)memo.slots * 32, stream);  // default policy: the memo lives for this launch only
    if (e != cudaSuccess) return e;
  }
  return dev.small_vocab ? launch_plan<true>(plan, a) : launch_plan<false>(plan, a);
}

}  // namespace xllm
