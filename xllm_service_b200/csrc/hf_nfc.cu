// hf_nfc.cu — exact NFC verification of requests for HF tokenizers with `normalizer: NFC` (Qwen2 / Qwen2.5 / Qwen3).
//
// The tokenizer kernels never normalise: a request is tokenised as is only when NFC provably leaves it unchanged.
// By default that proof is "every char is NFC-inert" (hf_pretok.cuh phase A), which refuses most text in scripts that
// need combining marks even when it is in NFC.  Under xllm_set_nfc_policy(h, XLLM_NFC_VERIFY) this kernel runs ahead
// of the tokenizer kernels and decides it exactly (UAX #15 quick check, completed where it answers "maybe"):
//   boundary char = canonical combining class (ccc) 0 and NFC_Quick_Check Yes (every ASCII byte is one);
//   chunk = a boundary char, or the start of the text, followed by the maximal run of non-boundary chars.
//   A text is in NFC iff (1) no char has NFC_QC = No, (2) no two adjacent chars a, b have ccc(a) > ccc(b) > 0, and
//   (3) every chunk that holds an NFC_QC = Maybe char is left unchanged by NFC (decomposition, canonical reordering,
//   composition — computed here for that chunk alone; NFC never reorders or composes across a boundary char).
// Such a chunk longer than kNfcChunkCap code points is refused even if it is in NFC; rules 1 and 2 are pairwise and
// have no cap.  Tables: scripts/gen_unicode_nfc.py -> unicode_nfc.inc (uploaded by SpDeviceModel::upload).
//
// One warp per request over a persistent grid (atomic task counter).  The warp reads the text as aligned 16-byte
// loads, 512 bytes per window; a window that is all ASCII is skipped after one vote.  In other windows every lane
// decodes the chars that start in its 16 bytes (the strict rules of utf8_unit, sp_encode.cu), looks up {ccc, QC} and
// applies rules 1 and 2; the previous char's ccc is carried across lanes and windows.  Rule 3 is the cold path: lane
// 0 walks back from the Maybe char to its chunk's start through global memory (bounded by the cap, so it may cross
// windows), forward to its end, and normalises the chunk in the warp's shared scratch.
// Verdict per request: 0 in NFC, 1 not in NFC (or a Maybe chunk over the cap), 2 malformed UTF-8.  Malformed input
// wins: after the first NFC violation the warp only keeps validating UTF-8, and stops at the first malformed byte.
#include "common.cuh"
#include "sp_encode.cuh"

namespace xllm {

namespace {

constexpr uint32_t kNfcFull = 0xffffffffu;
constexpr uint32_t kQcMaybe = 1, kQcNo = 2;
constexpr int kNfcDecompMax = kNfcChunkCap * 4;   // a full canonical decomposition is at most 4 code points

struct NfcScratch {
  uint32_t src[kNfcChunkCap];   // the chunk as it is
  uint32_t buf[kNfcDecompMax];  // cp | ccc << 21: decomposed, reordered, then composed in place
};

// {ccc (bits 0-7), NFC_Quick_Check (bits 8-9)} of a code point
__device__ __forceinline__ uint32_t nfc_prop(const SpDev& T, uint32_t cp) {
  if (cp < 0x80) return 0;
  return __ldg(T.nfc2 + (uint32_t)__ldg(T.nfc1 + (cp >> 8)) * 256u + (cp & 255u));
}
__device__ __forceinline__ bool nfc_boundary(uint32_t prop) { return prop == 0; }   // ccc 0 and QC Yes

// Strict UTF-8 at s[i] (s[0..n) is the request): the rules of utf8_unit (sp_encode.cu).  Returns the byte length,
// 0 if malformed; *cp = the code point.
__device__ __forceinline__ int nfc_decode(const uint8_t* s, int64_t i, int64_t n, uint32_t* cp) {
  const uint32_t b0 = s[i];
  if (b0 < 0x80) { *cp = b0; return 1; }
  auto trail = [](uint32_t x) { return (x & 0xC0u) == 0x80u; };
  const int64_t avail = n - i;
  if (avail >= 2 && (b0 & 0xE0u) == 0xC0u) {
    const uint32_t b1 = s[i + 1];
    const uint32_t c = ((b0 & 0x1Fu) << 6) | (b1 & 0x3Fu);
    if (trail(b1) && c >= 0x80) { *cp = c; return 2; }
  } else if (avail >= 3 && (b0 & 0xF0u) == 0xE0u) {
    const uint32_t b1 = s[i + 1], b2 = s[i + 2];
    const uint32_t c = ((b0 & 0x0Fu) << 12) | ((b1 & 0x3Fu) << 6) | (b2 & 0x3Fu);
    if (trail(b1) && trail(b2) && c >= 0x800 && !(c >= 0xD800 && c < 0xE000)) { *cp = c; return 3; }
  } else if (avail >= 4 && (b0 & 0xF8u) == 0xF0u) {
    const uint32_t b1 = s[i + 1], b2 = s[i + 2], b3 = s[i + 3];
    const uint32_t c = ((b0 & 0x07u) << 18) | ((b1 & 0x3Fu) << 12) | ((b2 & 0x3Fu) << 6) | (b3 & 0x3Fu);
    if (trail(b1) && trail(b2) && trail(b3) && c >= 0x10000 && c <= 0x10FFFF) { *cp = c; return 4; }
  }
  return 0;
}

constexpr uint32_t kSBase = 0xAC00, kLBase = 0x1100, kVBase = 0x1161, kTBase = 0x11A7;
constexpr uint32_t kLCount = 19, kVCount = 21, kTCount = 28, kNCount = kVCount * kTCount, kSCount = kLCount * kNCount;

// Appends the full canonical decomposition of cp (with each part's ccc) to buf[*m]; false when it does not fit.
__device__ bool nfc_decompose(const SpDev& T, uint32_t cp, uint32_t* buf, int* m) {
  uint32_t part[4];
  int k = 0;
  if (cp - kSBase < kSCount) {   // Hangul syllable: L V (T), all ccc 0
    const uint32_t si = cp - kSBase;
    part[k++] = kLBase + si / kNCount;
    part[k++] = kVBase + (si % kNCount) / kTCount;
    if (si % kTCount) part[k++] = kTBase + si % kTCount;
  } else {
    int lo = 0, hi = (int)T.n_nfc_decomp;
    if (cp >= 0xC0) {
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(T.nfc_decomp_cp + mid) < cp) lo = mid + 1;
        else hi = mid;
      }
    } else {
      lo = hi;
    }
    if (lo < (int)T.n_nfc_decomp && __ldg(T.nfc_decomp_cp + lo) == cp) {
      for (int j = 0; j < 4; ++j) {
        const uint32_t d = __ldg(T.nfc_decomp + 4 * lo + j);
        if (d) part[k++] = d;
      }
    } else {
      part[k++] = cp;
    }
  }
  if (*m + k > kNfcDecompMax) return false;
  for (int j = 0; j < k; ++j) buf[(*m)++] = part[j] | (nfc_prop(T, part[j]) & 0xFFu) << 21;
  return true;
}

// The primary composite of (a, b), or 0.
__device__ uint32_t nfc_compose(const SpDev& T, uint32_t a, uint32_t b) {
  if (a - kLBase < kLCount && b - kVBase < kVCount) return kSBase + ((a - kLBase) * kVCount + (b - kVBase)) * kTCount;
  if (a - kSBase < kSCount && (a - kSBase) % kTCount == 0 && b - kTBase - 1 < kTCount - 1) return a + (b - kTBase);
  const unsigned long long key = (unsigned long long)a << 21 | b;
  int lo = 0, hi = (int)T.n_nfc_comp;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(T.nfc_comp_key + mid) < key) lo = mid + 1;
    else hi = mid;
  }
  return (lo < (int)T.n_nfc_comp && __ldg(T.nfc_comp_key + lo) == key) ? __ldg(T.nfc_comp + lo) : 0u;
}

// Rule 3 for the Maybe char at s[i] (one lane).  Returns true when its chunk is left unchanged by NFC and has at most
// kNfcChunkCap code points; *chunk_end = the byte after the chunk.  Every byte before s[i] has been validated; a
// malformed byte ahead ends the chunk (the window scan refuses the request for it anyway).
__device__ bool nfc_chunk_ok(const SpDev& T, const uint8_t* s, int64_t n, int64_t i, NfcScratch& sc,
                             int64_t* chunk_end) {
  // back to the chunk's start: the nearest boundary char before s[i], or the start of the text
  int64_t st = i;
  int count = 1;
  while (st > 0) {
    int64_t p = st - 1;
    while (p > 0 && (s[p] & 0xC0u) == 0x80u) --p;
    uint32_t cp;
    nfc_decode(s, p, n, &cp);
    if (++count > kNfcChunkCap) return false;
    st = p;
    if (nfc_boundary(nfc_prop(T, cp))) break;
  }
  // forward to its end: the next boundary char (or the end of the text)
  uint32_t cp;
  int64_t en = i + nfc_decode(s, i, n, &cp);
  while (en < n) {
    const int l = nfc_decode(s, en, n, &cp);
    if (l == 0 || nfc_boundary(nfc_prop(T, cp))) break;
    if (++count > kNfcChunkCap) return false;
    en += l;
  }
  *chunk_end = en;
  // decompose, remembering the chunk as it is
  int nsrc = 0, m = 0;
  for (int64_t p = st; p < en;) {
    p += nfc_decode(s, p, n, &cp);
    sc.src[nsrc++] = cp;
    if (!nfc_decompose(T, cp, sc.buf, &m)) return false;
  }
  // canonical reordering: a stable sort of every run of non-starters by ccc
  for (int j = 1; j < m; ++j) {
    const uint32_t x = sc.buf[j], cx = x >> 21;
    if (cx == 0) continue;
    int k = j;
    while (k > 0 && (sc.buf[k - 1] >> 21) > cx) { sc.buf[k] = sc.buf[k - 1]; --k; }
    sc.buf[k] = x;
  }
  // canonical composition: a char composes with the last starter unless a char between them has ccc 0 or >= its own
  int out = 0, starter = -1;
  for (int j = 0; j < m; ++j) {
    const uint32_t x = sc.buf[j], c = x & 0x1FFFFFu, cc = x >> 21;
    if (starter >= 0) {
      const uint32_t last_cc = sc.buf[out - 1] >> 21;
      const bool blocked = out - 1 > starter && (last_cc == 0 || last_cc >= cc);
      if (!blocked) {
        const uint32_t comp = nfc_compose(T, sc.buf[starter] & 0x1FFFFFu, c);
        if (comp) { sc.buf[starter] = comp; continue; }   // a primary composite is a starter (ccc 0)
      }
    }
    if (cc == 0) starter = out;
    sc.buf[out++] = x;
  }
  if (out != nsrc) return false;
  for (int j = 0; j < out; ++j)
    if ((sc.buf[j] & 0x1FFFFFu) != sc.src[j]) return false;
  return true;
}

// 32-bit word j (bytes 4j .. 4j + 3) of a 16-byte block: mask of the bytes in [lo, hi)
__device__ __forceinline__ uint32_t nfc_word_mask(int j, int lo, int hi) {
  const int a = max(lo - 4 * j, 0), b = min(hi - 4 * j, 4);
  if (b <= a) return 0u;
  return (b - a == 4 ? 0xFFFFFFFFu : ((1u << (8 * (b - a))) - 1u)) << (8 * a);
}

__global__ void __launch_bounds__(kNfcWarps * 32, 8) hf_nfc_verify_kernel(
    const uint8_t* __restrict__ text, const int64_t* __restrict__ offsets, int n_req, uint8_t* __restrict__ verdict,
    unsigned int* __restrict__ task_counter, const __grid_constant__ SpDev T) {
  __shared__ NfcScratch scratch[kNfcWarps];
  NfcScratch& sc = scratch[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  for (;;) {
    unsigned int r = 0;
    if (lane == 0) r = atomicAdd(task_counter, 1u);
    r = __shfl_sync(kNfcFull, r, 0);
    if (r >= (unsigned)n_req) break;
    const int64_t beg = offsets[r];
    const int64_t n = offsets[r + 1] - beg;
    const uint8_t* s = text + beg;
    // aligned 16-byte blocks covering s[0..n): the first one starts `head` bytes before s (loads never leave the
    // aligned blocks that hold the request's bytes)
    const int head = (int)(reinterpret_cast<uintptr_t>(s) & 15u);
    const uint8_t* al = s - head;
    int v = 0;                  // 0 NFC so far, 1 not NFC (still validating UTF-8), 2 malformed
    uint32_t prev_ccc = 0;      // ccc of the last char before the window
    int64_t checked_to = 0;     // rule 3: the Maybe chunks that end before this byte are verified
    for (int64_t wb = 0; wb < n + head && v != 2; wb += 512) {
      const int64_t lb = wb + 16 * lane;          // this lane's block, in bytes from al
      const int lo = (int)max((int64_t)0, (int64_t)head - lb), hi = (int)min((int64_t)16, n + head - lb);
      uint32_t nonascii = 0;
      if (hi > lo) {
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(al + lb));
        nonascii = ((q.x & nfc_word_mask(0, lo, hi)) | (q.y & nfc_word_mask(1, lo, hi)) |
                    (q.z & nfc_word_mask(2, lo, hi)) | (q.w & nfc_word_mask(3, lo, hi))) & 0x80808080u;
      }
      if (!__any_sync(kNfcFull, nonascii != 0)) {
        prev_ccc = 0;
        continue;
      }
      // decode the chars that start in this lane's bytes: rules 1 and 2 inside the lane, UTF-8 validation
      bool bad = false, nfc_bad = false, has = false;
      uint32_t first_ccc = 0, last_ccc = 0, maybe = 0;   // maybe: bit k = a Maybe char starts at byte k
      for (int k = lo; k < hi; ++k) {
        const int64_t i = lb + k - head;
        const uint32_t b = s[i];
        uint32_t prop = 0;
        if ((b & 0xC0u) == 0x80u) {   // continuation byte: must belong to a lead byte at most 3 back
          bool cov = false;
          for (int d = 1; d <= 3 && i - d >= 0; ++d) {
            const uint32_t x = s[i - d];
            if ((x & 0xC0u) == 0x80u) continue;
            cov = (x >= 0xF0 ? 4 : (x >= 0xE0 ? 3 : (x >= 0xC0 ? 2 : 1))) > d;
            break;
          }
          bad |= !cov;
          continue;
        }
        if (b >= 0x80) {
          uint32_t cp;
          if (nfc_decode(s, i, n, &cp) == 0) { bad = true; continue; }
          prop = nfc_prop(T, cp);
        }
        const uint32_t ccc = prop & 0xFFu, qc = prop >> 8;
        nfc_bad |= qc == kQcNo;
        if (qc == kQcMaybe) maybe |= 1u << k;
        if (has) nfc_bad |= last_ccc > ccc && ccc > 0;
        else first_ccc = ccc;
        has = true;
        last_ccc = ccc;
      }
      // rule 2 across lanes: the previous char is the last one of the nearest lower lane that has one
      const uint32_t m_has = __ballot_sync(kNfcFull, has);
      const uint32_t lower = m_has & ((1u << lane) - 1u);
      const uint32_t from_lower = __shfl_sync(kNfcFull, last_ccc, lower ? 31 - __clz(lower) : 0);
      const uint32_t in_ccc = lower ? from_lower : prev_ccc;
      nfc_bad |= has && in_ccc > first_ccc && first_ccc > 0;
      const uint32_t top = __shfl_sync(kNfcFull, last_ccc, m_has ? 31 - __clz(m_has) : 0);
      if (m_has) prev_ccc = top;
      if (__any_sync(kNfcFull, bad)) { v = 2; break; }
      if (v != 0) continue;
      if (__any_sync(kNfcFull, nfc_bad)) { v = 1; continue; }
      // rule 3: every chunk that holds a Maybe char, in text order, each once
      uint32_t m_maybe = __ballot_sync(kNfcFull, maybe != 0);
      while (m_maybe && v == 0) {
        const int src = __ffs(m_maybe) - 1;
        m_maybe &= m_maybe - 1;
        uint32_t bits = __shfl_sync(kNfcFull, maybe, src);
        while (bits) {
          const int k = __ffs(bits) - 1;
          bits &= bits - 1;
          const int64_t i = wb + 16 * src + k - head;
          if (i < checked_to) continue;
          int ok = 0;
          long long end = 0;
          if (lane == 0) {
            int64_t e = 0;
            ok = nfc_chunk_ok(T, s, n, i, sc, &e) ? 1 : 0;
            end = e;
          }
          __syncwarp();
          ok = __shfl_sync(kNfcFull, ok, 0);
          end = __shfl_sync(kNfcFull, end, 0);
          if (!ok) { v = 1; break; }
          checked_to = end;
        }
      }
    }
    if (lane == 0) verdict[r] = (uint8_t)v;
  }
}

}  // namespace

cudaError_t hf_nfc_verify_launch(const SpDev& dev, const uint8_t* text, const int64_t* offsets, int n_req,
                                 uint8_t* verdict, unsigned int* task_counter, int blocks, cudaStream_t stream) {
  if (n_req <= 0 || blocks <= 0) return cudaSuccess;
  hf_nfc_verify_kernel<<<blocks, kNfcWarps * 32, 0, stream>>>(text, offsets, n_req, verdict, task_counter, dev);
  return cudaGetLastError();
}

}  // namespace xllm
