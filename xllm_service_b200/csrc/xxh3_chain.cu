// xxh3_chain.cu — chained per-block XXH3-128 over token-ID streams, sm_90a.
//
// Reference semantics (bit-exact target):
//   xllm_service/common/hash_util.cpp:18-45            xxh3_128bits_hash
//   xllm_service/scheduler/managers/global_kvcache_mgr.cpp:76-94   the per-request chain
//
// Fast path (block_size == 128, the reference default, global_gflags.cpp:114-116):
//   frame(b=0) = 512 B of tokens;  frame(b>0) = prev16 || 512 B of tokens = 528 B.
//   Both are XXH3's "long" class with <= 1024 B, so no scramble ever runs and the
//   8 x u64 accumulator is a plain wrap-around sum of per-stripe terms.  Only lanes
//   0,1 of stripe 0 see the previous key, so everything that touches HBM is
//   independent of the chain.
//
// Mapping: one warp owns 32 requests, LANE = REQUEST.  Per chain step b the warp
//   (1) stages block b of its 32 requests into shared memory with coalesced
//       16-byte cp.async (each warp-wide copy is one request's 512 contiguous bytes),
//       double/triple buffered so HBM latency is covered by the steps in flight;
//   (2) every lane folds its own request's 512 B out of shared memory (row stride
//       528 B => 128-bit LDS are bank-conflict free) into 8 accumulators;
//   (3) every lane adds the 2 prev-key terms, runs mergeAccs x2 + avalanche and
//       keeps the key in registers for step b+1 — 32 independent chains per warp, so
//       the serial part is fully SIMT-parallel;
//   (4) keys are staged [32 rows][8 keys] in shared memory and flushed as full
//       128-byte lines.
// Algorithmic HBM traffic: 512 B read + 16 B written per block (= 528 B/block).
//
// Generic path (any block_size in [1, 251], any alignment): one thread per
// request, frame built in local memory, all four XXH3 length classes.
#include "xxh3_chain.cuh"

#include <string.h>

#include "common.cuh"

namespace xllm {

namespace {

constexpr uint64_t P32_1 = 0x9E3779B1ULL;
constexpr uint64_t P32_2 = 0x85EBCA77ULL;
constexpr uint64_t P32_3 = 0xC2B2AE3DULL;
constexpr uint64_t P64_1 = 0x9E3779B185EBCA87ULL;
constexpr uint64_t P64_2 = 0xC2B2AE3D27D4EB4FULL;
constexpr uint64_t P64_3 = 0x165667B19E3779F9ULL;
constexpr uint64_t P64_4 = 0x85EBCA77C2B2AE63ULL;
constexpr uint64_t P64_5 = 0x27D4EB2F165667C5ULL;
constexpr uint64_t PRIME_MX1 = 0x165667919E3779F9ULL;
constexpr uint64_t PRIME_MX2 = 0x9FB21C651E98DF25ULL;

const uint8_t kSecretHost[192] = {
    0xb8, 0xfe, 0x6c, 0x39, 0x23, 0xa4, 0x4b, 0xbe, 0x7c, 0x01, 0x81, 0x2c, 0xf7, 0x21, 0xad, 0x1c,
    0xde, 0xd4, 0x6d, 0xe9, 0x83, 0x90, 0x97, 0xdb, 0x72, 0x40, 0xa4, 0xa4, 0xb7, 0xb3, 0x67, 0x1f,
    0xcb, 0x79, 0xe6, 0x4e, 0xcc, 0xc0, 0xe5, 0x78, 0x82, 0x5a, 0xd0, 0x7d, 0xcc, 0xff, 0x72, 0x21,
    0xb8, 0x08, 0x46, 0x74, 0xf7, 0x43, 0x24, 0x8e, 0xe0, 0x35, 0x90, 0xe6, 0x81, 0x3a, 0x26, 0x4c,
    0x3c, 0x28, 0x52, 0xbb, 0x91, 0xc3, 0x00, 0xcb, 0x88, 0xd0, 0x65, 0x8b, 0x1b, 0x53, 0x2e, 0xa3,
    0x71, 0x64, 0x48, 0x97, 0xa2, 0x0d, 0xf9, 0x4e, 0x38, 0x19, 0xef, 0x46, 0xa9, 0xde, 0xac, 0xd8,
    0xa8, 0xfa, 0x76, 0x3f, 0xe3, 0x9c, 0x34, 0x3f, 0xf9, 0xdc, 0xbb, 0xc7, 0xc7, 0x0b, 0x4f, 0x1d,
    0x8a, 0x51, 0xe0, 0x4b, 0xcd, 0xb4, 0x59, 0x31, 0xc8, 0x9f, 0x7e, 0xc9, 0xd9, 0x78, 0x73, 0x64,
    0xea, 0xc5, 0xac, 0x83, 0x34, 0xd3, 0xeb, 0xc3, 0xc5, 0x81, 0xa0, 0xff, 0xfa, 0x13, 0x63, 0xeb,
    0x17, 0x0d, 0xdd, 0x51, 0xb7, 0xf0, 0xda, 0x49, 0xd3, 0x16, 0x55, 0x26, 0x29, 0xd4, 0x68, 0x9e,
    0x2b, 0x16, 0xbe, 0x58, 0x7d, 0x47, 0xa1, 0xfc, 0x8f, 0xf8, 0xb8, 0xd1, 0x7a, 0xd0, 0x31, 0xce,
    0x45, 0xcb, 0x3a, 0x8f, 0x95, 0x16, 0x04, 0x28, 0xaf, 0xd7, 0xfb, 0xca, 0xbb, 0x4b, 0x40, 0x7e,
};

inline uint64_t host_rd64(const uint8_t* p) {
  uint64_t v;
  memcpy(&v, p, 8);
  return v;
}

// ------------------------------------------------------------------ device math
__device__ __forceinline__ uint64_t mul32x32(uint64_t v) {
  return (uint64_t)(uint32_t)v * (uint64_t)(uint32_t)(v >> 32);
}
__device__ __forceinline__ uint64_t mul128_fold64(uint64_t a, uint64_t b) {
  return (a * b) ^ __umul64hi(a, b);
}
__device__ __forceinline__ uint64_t xxh3_avalanche(uint64_t h) {
  h ^= h >> 37;
  h *= PRIME_MX1;
  h ^= h >> 32;
  return h;
}
__device__ __forceinline__ uint64_t xxh64_avalanche(uint64_t h) {
  h ^= h >> 33;
  h *= P64_2;
  h ^= h >> 29;
  h *= P64_3;
  h ^= h >> 32;
  return h;
}
__device__ __forceinline__ uint64_t u64_of(uint32_t lo, uint32_t hi) { return (uint64_t)lo | ((uint64_t)hi << 32); }

// ------------------------------------------------------------- fast path kernel
constexpr int kBlockTokens = 128;   // tokens per KV block on the fast path
constexpr int kRowsPerWarp = 32;    // lane == request
constexpr int kQuarterU4 = 8;       // pipeline unit: one 128-byte quarter of a block per row
constexpr int kQRowU4 = 9;          // padded row stride in the stage: 144 B => conflict-free LDS.128
constexpr int kKeyRowU4 = 9;        // 8 keys + 1 pad per row in the output stage
constexpr int kKeysPerFlush = 8;

template <int STAGES>
struct FastSmem {
  uint4 stage[STAGES][kRowsPerWarp * kQRowU4];  // STAGES x 4.5 KB
  uint4 keys[kRowsPerWarp * kKeyRowU4];         // 4.5 KB
  uint8_t* row_key[kRowsPerWarp];               // key base pointer of each row
  int32_t row_nb[kRowsPerWarp];                 // blocks in each row
  unsigned long long bar[STAGES];               // BULK: one mbarrier per stage (32 arrivals + the copies' bytes)
};

// ---- bulk-copy staging (XLLM_XXH3_BULK=1): every lane moves its own row's 128-byte quarter with one
// cp.async.bulk (the async proxy's copy engine instead of eight 16-byte LDGSTS issued by the warp); completion is
// counted in bytes on the stage's mbarrier
__device__ __forceinline__ void mbar_init(unsigned long long* b, unsigned count) {
  asm volatile("mbarrier.init.shared.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* b) {
  asm volatile("{ .reg .b64 st; mbarrier.arrive.shared.b64 st, [%0]; }" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect(unsigned long long* b, unsigned bytes) {
  asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared.b64 st, [%0], %1; }" ::"r"(smem_u32(b)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned parity) {
  asm volatile(
      "{ .reg .pred p;\n"
      "XLLM_MBAR_WAIT_%=: mbarrier.try_wait.parity.shared.b64 p, [%0], %1;\n"
      "@!p bra XLLM_MBAR_WAIT_%=; }"
      ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(b)) : "memory");
}

__device__ __forceinline__ uint4 lds128(const uint4* p) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "r"(smem_u32(p)));
  return v;
}

// acc[L ^ 1] += dv ; acc[L] += lo32(dv ^ key) * hi32(dv ^ key)
#define XXH_ROUND(L, DV, KEY)           \
  do {                                  \
    acc[(L) ^ 1] += (DV);               \
    acc[(L)] += mul32x32((DV) ^ (KEY)); \
  } while (0)

// Fold quarter QTR (token u64 16*QTR .. 16*QTR+15) of one 512-byte block into acc[8].
// CHAINED == false: frame u64 index f = j         (len 512: 7 full stripes + last stripe)
// CHAINED == true : frame u64 index f = j + 2     (len 528: 8 full stripes + last stripe)
// Full stripe k = f / 8 (only while f < 8 * nbStripes), lane l = f % 8, key s[k + l].
// Last stripe = token u64 56..63 (frame bytes len-64 .. len), lane j - 56, key last[j - 56].
template <int QTR, bool CHAINED>
__device__ __forceinline__ void fold_quarter(const uint4* row, const Xxh3Consts& C, uint64_t (&acc)[8]) {
  uint4 v[kQuarterU4];
#pragma unroll
  for (int q = 0; q < kQuarterU4; ++q) v[q] = lds128(row + q);
#pragma unroll
  for (int q = 0; q < kQuarterU4; ++q) {
    const uint64_t d0 = u64_of(v[q].x, v[q].y);
    const uint64_t d1 = u64_of(v[q].z, v[q].w);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = 16 * QTR + 2 * q + h;
      const uint64_t dv = h ? d1 : d0;
      const int f = CHAINED ? j + 2 : j;
      const int full_limit = CHAINED ? 64 : 56;
      if (f < full_limit) {
        const int k = f >> 3, l = f & 7;
        XXH_ROUND(l, dv, C.s[k + l]);
      }
      if (j >= 56) {
        const int l = j - 56;
        XXH_ROUND(l, dv, C.last[l]);
      }
    }
  }
}

__device__ __forceinline__ void finish_block(uint64_t (&acc)[8], const Xxh3Consts& C, uint64_t len, uint64_t& lo,
                                             uint64_t& hi) {
  uint64_t rl = len * P64_1;
  uint64_t rh = ~(len * P64_2);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    rl += mul128_fold64(acc[2 * i] ^ C.mlo[2 * i], acc[2 * i + 1] ^ C.mlo[2 * i + 1]);
    rh += mul128_fold64(acc[2 * i] ^ C.mhi[2 * i], acc[2 * i + 1] ^ C.mhi[2 * i + 1]);
  }
  lo = xxh3_avalanche(rl);
  hi = xxh3_avalanche(rh);
}

template <int STAGES, bool BULK = false>
__global__ void __launch_bounds__(32) xxh3_chain128_kernel(const int32_t* __restrict__ tokens,
                                                           const int64_t* __restrict__ tok_start,
                                                           const int32_t* __restrict__ n_tok,
                                                           uint8_t* __restrict__ keys,
                                                           const int64_t* __restrict__ key_start, int n_req,
                                                           const __grid_constant__ Xxh3Consts C,
                                                           unsigned int* __restrict__ task_counter) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FastSmem<STAGES>& sm = *reinterpret_cast<FastSmem<STAGES>*>(smem_raw);
  const int lane = threadIdx.x;
  const int n_tasks = (n_req + kRowsPerWarp - 1) / kRowsPerWarp;
  const int piece = lane & 7;   // which 16 B of a row's 128-byte quarter this lane copies
  const int rsub = lane >> 3;   // copies cover 4 rows per instruction: row = 4 * it + rsub
  // BULK: stage / phase of the next unit to issue and to consume (issued == consumed at every task boundary)
  int b_islot = 0, b_cslot = 0;
  unsigned b_ipar = 0, b_cpar = 0;
  if constexpr (BULK) {
    if (lane == 0) {
      for (int i = 0; i < STAGES; ++i) mbar_init(&sm.bar[i], 32);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
  }

  for (;;) {
    unsigned int task = 0;
    if (lane == 0) task = atomicAdd(task_counter, 1u);
    task = __shfl_sync(0xffffffffu, task, 0);
    if (task >= (unsigned)n_tasks) break;

    const int r = (int)task * kRowsPerWarp + lane;
    const bool valid = r < n_req;
    const int my_nb = valid ? (n_tok[r] / kBlockTokens) : 0;
    const int32_t* my_tok = valid ? tokens + tok_start[r] : tokens;
    sm.row_key[lane] = valid ? keys + 16 * key_start[r] : keys;
    sm.row_nb[lane] = my_nb;
    int max_nb = my_nb;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) max_nb = max(max_nb, __shfl_xor_sync(0xffffffffu, max_nb, o));

    // The 8 rows this lane copies for, kept in registers.
    const int32_t* cp_src[8];
    int cp_nb[8];
    unsigned int aligned_mask = 0;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int q = 4 * it + rsub;
      const unsigned long long p = __shfl_sync(0xffffffffu, (unsigned long long)my_tok, q);
      cp_src[it] = reinterpret_cast<const int32_t*>(p) + piece * 4;
      cp_nb[it] = __shfl_sync(0xffffffffu, my_nb, q);
      if ((p & 15ull) == 0) aligned_mask |= 1u << it;
    }
    __syncwarp();

    // Issue the copies of pipeline unit u = 4 * b + qtr into slot u % STAGES.
    auto issue = [&](int u, int slot) {
      const int b = u >> 2;
      if constexpr (BULK) {
        if (b < max_nb) {
          // lane == row: one 128-byte bulk copy when the row is 16-byte aligned, else the lane copies its quarter itself
          const int32_t* src = my_tok + b * kBlockTokens + (u & 3) * 32;
          uint4* dst = sm.stage[b_islot] + lane * kQRowU4;
          if (b >= my_nb) {
            mbar_arrive(&sm.bar[b_islot]);
          } else if ((reinterpret_cast<uintptr_t>(my_tok) & 15u) == 0) {
            mbar_arrive_expect(&sm.bar[b_islot], 128u);
            bulk_g2s(dst, src, 128u, &sm.bar[b_islot]);
          } else {
            uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
#pragma unroll 8
            for (int i = 0; i < 32; ++i) d32[i] = (uint32_t)__ldg(src + i);
            mbar_arrive(&sm.bar[b_islot]);
          }
          if (++b_islot == STAGES) { b_islot = 0; b_ipar ^= 1u; }
        }
        return;
      }
      if (b < max_nb) {
        uint4* st = sm.stage[slot] + rsub * kQRowU4 + piece;
        const int tok_off = b * kBlockTokens + (u & 3) * 32;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          if (b < cp_nb[it]) {
            const int32_t* src = cp_src[it] + tok_off;
            uint4* dst = st + it * 4 * kQRowU4;
            if (aligned_mask & (1u << it)) {
              cp_async_16(dst, src);
            } else {  // row not 16-byte aligned: same bytes, 4-byte copies
              cp_async_4(reinterpret_cast<uint32_t*>(dst) + 0, src + 0);
              cp_async_4(reinterpret_cast<uint32_t*>(dst) + 1, src + 1);
              cp_async_4(reinterpret_cast<uint32_t*>(dst) + 2, src + 2);
              cp_async_4(reinterpret_cast<uint32_t*>(dst) + 3, src + 3);
            }
          }
        }
      }
      cp_async_commit();  // always commit so group accounting stays uniform
    };

    int issue_slot = 0;
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
      issue(s, issue_slot);
      issue_slot = (issue_slot + 1 == STAGES) ? 0 : issue_slot + 1;
    }
    int slot = 0;

    uint64_t prev_lo = 0, prev_hi = 0;
    for (int b = 0; b < max_nb; ++b) {
      uint64_t acc[8] = {P32_3, P64_1, P64_2, P64_3, P64_4, P32_2, P64_5, P32_1};
      const bool active = b < my_nb;
#define XXH_STEP(QTR)                                                         \
  do {                                                                        \
    issue(4 * b + (QTR) + STAGES - 1, issue_slot);                            \
    issue_slot = (issue_slot + 1 == STAGES) ? 0 : issue_slot + 1;             \
    if constexpr (BULK) {                                                     \
      mbar_wait(&sm.bar[b_cslot], b_cpar);                                    \
      slot = b_cslot;                                                         \
      if (++b_cslot == STAGES) { b_cslot = 0; b_cpar ^= 1u; }                 \
    } else {                                                                  \
      cp_async_wait<STAGES - 1>();                                            \
    }                                                                         \
    __syncwarp();                                                             \
    if (active) {                                                             \
      const uint4* row = sm.stage[slot] + lane * kQRowU4;                     \
      if (b == 0) fold_quarter<QTR, false>(row, C, acc);                      \
      else fold_quarter<QTR, true>(row, C, acc);                              \
    }                                                                         \
    slot = (slot + 1 == STAGES) ? 0 : slot + 1;                               \
    __syncwarp(); /* the slot just consumed may be refilled by the next issue */ \
  } while (0)
      XXH_STEP(0);
      XXH_STEP(1);
      XXH_STEP(2);
      XXH_STEP(3);
#undef XXH_STEP

      if (active) {
        uint64_t lo, hi;
        if (b == 0) {
          finish_block(acc, C, 512, lo, hi);
        } else {
          XXH_ROUND(0, prev_lo, C.s[0]);  // stripe 0, lane 0 <- previous key low64
          XXH_ROUND(1, prev_hi, C.s[1]);  // stripe 0, lane 1 <- previous key high64
          finish_block(acc, C, 528, lo, hi);
        }
        prev_lo = lo;
        prev_hi = hi;
        sm.keys[lane * kKeyRowU4 + (b % kKeysPerFlush)] =
            make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
      }

      if ((b % kKeysPerFlush) == kKeysPerFlush - 1 || b == max_nb - 1) {
        __syncwarp();
        const int b0 = b - (b % kKeysPerFlush);
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int q = it * 4 + rsub;
          if (b0 + piece < sm.row_nb[q] && b0 + piece <= b) {
            reinterpret_cast<uint4*>(sm.row_key[q])[b0 + piece] = sm.keys[q * kKeyRowU4 + piece];
          }
        }
        __syncwarp();
      }
    }
    cp_async_wait<0>();
    __syncwarp();
  }
}

// ---------------------------------------------------------- generic path kernel
struct H128 {
  uint64_t lo, hi;
};
__device__ __forceinline__ uint64_t rd64(const uint8_t* p) {
  uint64_t v = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) v |= (uint64_t)p[i] << (8 * i);
  return v;
}
__device__ __forceinline__ uint32_t rd32(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }
__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
  return ((uint64_t)bswap32((uint32_t)x) << 32) | bswap32((uint32_t)(x >> 32));
}
__device__ __forceinline__ uint64_t mix16B(const uint8_t* in, const uint8_t* sec, uint64_t seed) {
  return mul128_fold64(rd64(in) ^ (rd64(sec) + seed), rd64(in + 8) ^ (rd64(sec + 8) - seed));
}
__device__ __forceinline__ H128 mix32B(H128 a, const uint8_t* i1, const uint8_t* i2, const uint8_t* sec,
                                       uint64_t seed) {
  a.lo += mix16B(i1, sec, seed);
  a.lo ^= rd64(i2) + rd64(i2 + 8);
  a.hi += mix16B(i2, sec + 16, seed);
  a.hi ^= rd64(i1) + rd64(i1 + 8);
  return a;
}
__device__ __forceinline__ H128 mid_finish(H128 a, uint64_t len, uint64_t seed) {
  H128 h;
  h.lo = xxh3_avalanche(a.lo + a.hi);
  h.hi = 0ULL - xxh3_avalanche(a.lo * P64_1 + a.hi * P64_4 + (len - seed) * P64_2);
  return h;
}

// Generic XXH3_128bits_withSeed over `len` bytes at `in` (any class).
__device__ H128 xxh3_128_generic(const uint8_t* in, uint32_t len, const Xxh3Consts& C) {
  const uint8_t* ks = C.ksecret;
  const uint64_t seed = C.seed;
  H128 h;
  if (len == 0) {
    h.lo = xxh64_avalanche(seed ^ (rd64(ks + 64) ^ rd64(ks + 72)));
    h.hi = xxh64_avalanche(seed ^ (rd64(ks + 80) ^ rd64(ks + 88)));
    return h;
  }
  if (len <= 3) {
    const uint8_t c1 = in[0], c2 = in[len >> 1], c3 = in[len - 1];
    const uint32_t cl = ((uint32_t)c1 << 16) | ((uint32_t)c2 << 24) | (uint32_t)c3 | (len << 8);
    const uint32_t sw = bswap32(cl);
    const uint32_t ch = (sw << 13) | (sw >> 19);
    const uint64_t fl = (uint64_t)(rd32(ks) ^ rd32(ks + 4)) + seed;
    const uint64_t fh = (uint64_t)(rd32(ks + 8) ^ rd32(ks + 12)) - seed;
    h.lo = xxh64_avalanche((uint64_t)cl ^ fl);
    h.hi = xxh64_avalanche((uint64_t)ch ^ fh);
    return h;
  }
  if (len <= 8) {
    const uint64_t s2 = seed ^ ((uint64_t)bswap32((uint32_t)seed) << 32);
    const uint64_t in64 = (uint64_t)rd32(in) + ((uint64_t)rd32(in + len - 4) << 32);
    const uint64_t keyed = in64 ^ ((rd64(ks + 16) ^ rd64(ks + 24)) + s2);
    const uint64_t m = P64_1 + ((uint64_t)len << 2);
    uint64_t mlo = keyed * m, mhi = __umul64hi(keyed, m);
    mhi += mlo << 1;
    mlo ^= mhi >> 3;
    mlo ^= mlo >> 35;
    mlo *= PRIME_MX2;
    mlo ^= mlo >> 28;
    h.lo = mlo;
    h.hi = xxh3_avalanche(mhi);
    return h;
  }
  if (len <= 16) {
    const uint64_t fl = (rd64(ks + 32) ^ rd64(ks + 40)) - seed;
    const uint64_t fh = (rd64(ks + 48) ^ rd64(ks + 56)) + seed;
    const uint64_t ilo = rd64(in);
    uint64_t ihi = rd64(in + len - 8);
    const uint64_t x = ilo ^ ihi ^ fl;
    uint64_t mlo = x * P64_1, mhi = __umul64hi(x, P64_1);
    mlo += (uint64_t)(len - 1) << 54;
    ihi ^= fh;
    mhi += ihi + (uint64_t)(uint32_t)ihi * (P32_2 - 1);
    mlo ^= bswap64(mhi);
    uint64_t hlo = mlo * P64_2, hhi = __umul64hi(mlo, P64_2);
    hhi += mhi * P64_2;
    h.lo = xxh3_avalanche(hlo);
    h.hi = xxh3_avalanche(hhi);
    return h;
  }
  if (len <= 128) {
    H128 a = {(uint64_t)len * P64_1, 0};
    if (len > 32) {
      if (len > 64) {
        if (len > 96) a = mix32B(a, in + 48, in + len - 64, ks + 96, seed);
        a = mix32B(a, in + 32, in + len - 48, ks + 64, seed);
      }
      a = mix32B(a, in + 16, in + len - 32, ks + 32, seed);
    }
    a = mix32B(a, in, in + len - 16, ks, seed);
    return mid_finish(a, len, seed);
  }
  if (len <= 240) {
    H128 a = {(uint64_t)len * P64_1, 0};
    uint32_t i;
    for (i = 32; i < 160; i += 32) a = mix32B(a, in + i - 32, in + i - 16, ks + i - 32, seed);
    a.lo = xxh3_avalanche(a.lo);
    a.hi = xxh3_avalanche(a.hi);
    for (i = 160; i <= len; i += 32) a = mix32B(a, in + i - 32, in + i - 16, ks + 3 + i - 160, seed);
    a = mix32B(a, in + len - 16, in + len - 32, ks + 136 - 17 - 16, 0ULL - seed);
    return mid_finish(a, len, seed);
  }
  // long class; the chain frame is < 1024 B (hash_util.cpp:33) so at most one partial
  // block, but the scramble is kept so the function is XXH3-complete.
  const uint8_t* sec = C.secret;
  uint64_t acc[8] = {P32_3, P64_1, P64_2, P64_3, P64_4, P32_2, P64_5, P32_1};
  const uint32_t nb_blocks = (len - 1) / 1024;
  for (uint32_t n = 0; n < nb_blocks; ++n) {
    for (uint32_t s = 0; s < 16; ++s)
      for (int l = 0; l < 8; ++l) {
        const uint64_t dv = rd64(in + n * 1024 + s * 64 + 8 * l);
        acc[l ^ 1] += dv;
        acc[l] += mul32x32(dv ^ rd64(sec + 8 * s + 8 * l));
      }
    for (int l = 0; l < 8; ++l) {
      uint64_t a = acc[l];
      a ^= a >> 47;
      a ^= rd64(sec + 128 + 8 * l);
      a *= P32_1;
      acc[l] = a;
    }
  }
  const uint32_t nb_stripes = ((len - 1) - 1024 * nb_blocks) / 64;
  for (uint32_t s = 0; s < nb_stripes; ++s)
    for (int l = 0; l < 8; ++l) {
      const uint64_t dv = rd64(in + nb_blocks * 1024 + s * 64 + 8 * l);
      acc[l ^ 1] += dv;
      acc[l] += mul32x32(dv ^ rd64(sec + 8 * s + 8 * l));
    }
  for (int l = 0; l < 8; ++l) {
    const uint64_t dv = rd64(in + len - 64 + 8 * l);
    acc[l ^ 1] += dv;
    acc[l] += mul32x32(dv ^ rd64(sec + 121 + 8 * l));
  }
  uint64_t rl = (uint64_t)len * P64_1, rh = ~((uint64_t)len * P64_2);
  for (int i = 0; i < 4; ++i) {
    rl += mul128_fold64(acc[2 * i] ^ rd64(sec + 11 + 16 * i), acc[2 * i + 1] ^ rd64(sec + 11 + 16 * i + 8));
    rh += mul128_fold64(acc[2 * i] ^ rd64(sec + 117 + 16 * i), acc[2 * i + 1] ^ rd64(sec + 117 + 16 * i + 8));
  }
  h.lo = xxh3_avalanche(rl);
  h.hi = xxh3_avalanche(rh);
  return h;
}

__global__ void __launch_bounds__(128) xxh3_chain_generic_kernel(const int32_t* __restrict__ tokens,
                                                                  const int64_t* __restrict__ tok_start,
                                                                  const int32_t* __restrict__ n_tok,
                                                                  uint8_t* __restrict__ keys,
                                                                  const int64_t* __restrict__ key_start, int n_req,
                                                                  int block_size,
                                                                  const __grid_constant__ Xxh3Consts C) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_req) return;
  const int32_t* tk = tokens + tok_start[r];
  uint8_t* out = keys + 16 * key_start[r];
  const int nb = n_tok[r] / block_size;
  uint8_t frame[1024];
  uint64_t plo = 0, phi = 0;
  for (int b = 0; b < nb; ++b) {
    uint32_t off = 0;
    if (b > 0) {
      for (int i = 0; i < 8; ++i) frame[i] = (uint8_t)(plo >> (8 * i));
      for (int i = 0; i < 8; ++i) frame[8 + i] = (uint8_t)(phi >> (8 * i));
      off = 16;
    }
    for (int t = 0; t < block_size; ++t) {
      const uint32_t v = (uint32_t)tk[(size_t)b * block_size + t];
      frame[off + 4 * t + 0] = (uint8_t)v;
      frame[off + 4 * t + 1] = (uint8_t)(v >> 8);
      frame[off + 4 * t + 2] = (uint8_t)(v >> 16);
      frame[off + 4 * t + 3] = (uint8_t)(v >> 24);
    }
    const H128 h = xxh3_128_generic(frame, off + 4u * (uint32_t)block_size, C);
    plo = h.lo;
    phi = h.hi;
    for (int i = 0; i < 8; ++i) out[16 * (size_t)b + i] = (uint8_t)(plo >> (8 * i));
    for (int i = 0; i < 8; ++i) out[16 * (size_t)b + 8 + i] = (uint8_t)(phi >> (8 * i));
  }
}

__global__ void xxh3_single_kernel(const uint8_t* __restrict__ data, uint32_t len, uint8_t* __restrict__ out16,
                                   const __grid_constant__ Xxh3Consts C) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const H128 h = xxh3_128_generic(data, len, C);
  for (int i = 0; i < 8; ++i) out16[i] = (uint8_t)(h.lo >> (8 * i));
  for (int i = 0; i < 8; ++i) out16[8 + i] = (uint8_t)(h.hi >> (8 * i));
}

constexpr int kFastStages = 3;

}  // namespace

void xxh3_make_consts(uint32_t seed32, Xxh3Consts* out) {
  const uint64_t seed = (uint64_t)seed32;
  uint8_t S[192];
  for (int i = 0; i < 12; ++i) {
    const uint64_t a = host_rd64(kSecretHost + 16 * i) + seed;
    const uint64_t b = host_rd64(kSecretHost + 16 * i + 8) - seed;
    memcpy(S + 16 * i, &a, 8);
    memcpy(S + 16 * i + 8, &b, 8);
  }
  for (int i = 0; i < 16; ++i) out->s[i] = host_rd64(S + 8 * i);
  for (int i = 0; i < 8; ++i) out->last[i] = host_rd64(S + 121 + 8 * i);
  for (int i = 0; i < 8; ++i) out->mlo[i] = host_rd64(S + 11 + 8 * i);
  for (int i = 0; i < 8; ++i) out->mhi[i] = host_rd64(S + 117 + 8 * i);
  out->seed = seed;
  memcpy(out->secret, S, 192);
  memcpy(out->ksecret, kSecretHost, 192);
}

cudaError_t xxh3_single_launch(const uint8_t* d_data, size_t len, uint8_t* d_out16, const Xxh3Consts& consts,
                               cudaStream_t stream) {
  if (len > 0xFFFFFFFFull) return cudaErrorInvalidValue;
  xxh3_single_kernel<<<1, 32, 0, stream>>>(d_data, (uint32_t)len, d_out16, consts);
  return cudaGetLastError();
}

cudaError_t xxh3_chain_launch(const int32_t* tokens, const int64_t* tok_start, const int32_t* n_tok, uint8_t* keys,
                              const int64_t* key_start, int n_req, int block_size, const Xxh3Consts& consts,
                              unsigned int* task_counter, cudaStream_t stream) {
  if (n_req <= 0) return cudaSuccess;
  if (block_size == kBlockTokens) {
    static DeviceOnce once;
    const size_t smem = sizeof(FastSmem<kFastStages>);
    cudaError_t e0 = cudaSuccess;
    const int n_sm = once.get(
        [&] {
          cudaError_t r = cudaFuncSetAttribute(xxh3_chain128_kernel<kFastStages, true>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
          if (r != cudaSuccess) return r;
          return cudaFuncSetAttribute(xxh3_chain128_kernel<kFastStages>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        },
        &e0);
    if (e0 != cudaSuccess) return e0;
    cudaError_t e = cudaMemsetAsync(task_counter, 0, sizeof(unsigned int), stream);
    if (e != cudaSuccess) return e;
    const int n_tasks = (n_req + kRowsPerWarp - 1) / kRowsPerWarp;
    int warps_per_sm = (int)((227 * 1024) / (smem + 1024));
    if (warps_per_sm > 16) warps_per_sm = 16;
    // Balanced persistent grid: every warp runs the same number of 32-request tasks.
    const int max_warps = n_sm * warps_per_sm;
    const int rounds = (n_tasks + max_warps - 1) / max_warps;
    int grid = (n_tasks + rounds - 1) / rounds;
    static const bool bulk = [] { const char* w = getenv("XLLM_XXH3_BULK"); return w && atoi(w) != 0; }();
    if (bulk)
      xxh3_chain128_kernel<kFastStages, true><<<grid, 32, smem, stream>>>(tokens, tok_start, n_tok, keys, key_start,
                                                                          n_req, consts, task_counter);
    else
      xxh3_chain128_kernel<kFastStages><<<grid, 32, smem, stream>>>(tokens, tok_start, n_tok, keys, key_start, n_req,
                                                                    consts, task_counter);
    return cudaGetLastError();
  }
  const int threads = 128;
  const int grid = (n_req + threads - 1) / threads;
  xxh3_chain_generic_kernel<<<grid, threads, 0, stream>>>(tokens, tok_start, n_tok, keys, key_start, n_req,
                                                          block_size, consts);
  return cudaGetLastError();
}

}  // namespace xllm
