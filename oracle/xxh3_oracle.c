/*
 * oracle/xxh3_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Scalar CPU restatement of the block-hash step of the reference's prefix-cache
 * path.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this; the product (libxllm_ingest.so) never
 * links or calls it.
 *
 * What it restates
 *   - xllm_service/common/hash_util.cpp:18-45   xxh3_128bits_hash(prev, tokens, out)
 *       prev == NULL : H = XXH3_128bits_withSeed(tokens, 4*n, seed)
 *       prev != NULL : H = XXH3_128bits_withSeed(prev16 || tokens, 16 + 4*n, seed)
 *                      (1024-byte stack frame, CHECK_GT(1024, len): hash_util.cpp:29-33)
 *       out = memcpy of XXH128_hash_t  = low64 LE || high64 LE  (hash_util.cpp:26-27,42-43)
 *   - xllm_service/scheduler/managers/global_kvcache_mgr.cpp:76-94  the per-request
 *       chain: floor(n/block_size) blocks, block 0 unchained, block i>0 chained on
 *       the previous key (prev and out alias).
 *   - seed: FLAGS_xxh3_128bits_seed, uint32 default 1024 (global_gflags.cpp:60),
 *       zero-extended to XXH64_hash_t.
 *
 * Third-party arithmetic: xxHash (submodule third_party/xxHash @ ce037363, absent
 * from the reference checkout).  XXH3 output is frozen since v0.8.0; this file restates
 * the published algorithm (all four length classes + the long path with scramble)
 * and is pinned against libxxhash.so.0.8.2 and the vendored xxhash.h v0.8.3 by
 * tests/test_oracle_xxh3.py and the committed vectors in tests/golden/xxh3_kat.json.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#define P32_1 0x9E3779B1U
#define P32_2 0x85EBCA77U
#define P32_3 0xC2B2AE3DU
#define P64_1 0x9E3779B185EBCA87ULL
#define P64_2 0xC2B2AE3D27D4EB4FULL
#define P64_3 0x165667B19E3779F9ULL
#define P64_4 0x85EBCA77C2B2AE63ULL
#define P64_5 0x27D4EB2F165667C5ULL
#define PRIME_MX1 0x165667919E3779F9ULL
#define PRIME_MX2 0x9FB21C651E98DF25ULL

#define SECRET_SIZE 192
#define STRIPE_LEN 64
#define SECRET_CONSUME_RATE 8
#define SECRET_MERGEACCS_START 11
#define SECRET_LASTACC_START 7
#define SECRET_SIZE_MIN 136
#define MIDSIZE_MAX 240
#define MIDSIZE_STARTOFFSET 3
#define MIDSIZE_LASTOFFSET 17

static const uint8_t kSecret[SECRET_SIZE] = {
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

typedef struct { uint64_t low64, high64; } h128_t;

static inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; } /* LE host */
static inline uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline void wr64(uint8_t* p, uint64_t v) { memcpy(p, &v, 8); }
static inline uint32_t swap32(uint32_t x) { return __builtin_bswap32(x); }
static inline uint64_t swap64(uint64_t x) { return __builtin_bswap64(x); }
static inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

static inline h128_t mult64to128(uint64_t a, uint64_t b) {
  __uint128_t p = (__uint128_t)a * b;
  h128_t r = {(uint64_t)p, (uint64_t)(p >> 64)};
  return r;
}
static inline uint64_t mul128_fold64(uint64_t a, uint64_t b) {
  h128_t p = mult64to128(a, b);
  return p.low64 ^ p.high64;
}
static inline uint64_t xorshift64(uint64_t v, int s) { return v ^ (v >> s); }
static inline uint64_t xxh3_avalanche(uint64_t h) {
  h = xorshift64(h, 37); h *= PRIME_MX1; h = xorshift64(h, 32); return h;
}
static inline uint64_t xxh64_avalanche(uint64_t h) {
  h ^= h >> 33; h *= P64_2; h ^= h >> 29; h *= P64_3; h ^= h >> 32; return h;
}

/* ---- len <= 16 ---- */
static h128_t len_1to3(const uint8_t* in, size_t len, const uint8_t* sec, uint64_t seed) {
  uint8_t c1 = in[0], c2 = in[len >> 1], c3 = in[len - 1];
  uint32_t combl = ((uint32_t)c1 << 16) | ((uint32_t)c2 << 24) | (uint32_t)c3 | ((uint32_t)len << 8);
  uint32_t combh = rotl32(swap32(combl), 13);
  uint64_t flipl = (uint64_t)(rd32(sec) ^ rd32(sec + 4)) + seed;
  uint64_t fliph = (uint64_t)(rd32(sec + 8) ^ rd32(sec + 12)) - seed;
  h128_t h = {xxh64_avalanche((uint64_t)combl ^ flipl), xxh64_avalanche((uint64_t)combh ^ fliph)};
  return h;
}
static h128_t len_4to8(const uint8_t* in, size_t len, const uint8_t* sec, uint64_t seed) {
  seed ^= (uint64_t)swap32((uint32_t)seed) << 32;
  uint32_t lo = rd32(in), hi = rd32(in + len - 4);
  uint64_t in64 = lo + ((uint64_t)hi << 32);
  uint64_t flip = (rd64(sec + 16) ^ rd64(sec + 24)) + seed;
  h128_t m = mult64to128(in64 ^ flip, P64_1 + ((uint64_t)len << 2));
  m.high64 += m.low64 << 1;
  m.low64 ^= m.high64 >> 3;
  m.low64 = xorshift64(m.low64, 35);
  m.low64 *= PRIME_MX2;
  m.low64 = xorshift64(m.low64, 28);
  m.high64 = xxh3_avalanche(m.high64);
  return m;
}
static h128_t len_9to16(const uint8_t* in, size_t len, const uint8_t* sec, uint64_t seed) {
  uint64_t flipl = (rd64(sec + 32) ^ rd64(sec + 40)) - seed;
  uint64_t fliph = (rd64(sec + 48) ^ rd64(sec + 56)) + seed;
  uint64_t ilo = rd64(in), ihi = rd64(in + len - 8);
  h128_t m = mult64to128(ilo ^ ihi ^ flipl, P64_1);
  m.low64 += (uint64_t)(len - 1) << 54;
  ihi ^= fliph;
  m.high64 += ihi + (uint64_t)(uint32_t)ihi * (uint64_t)(P32_2 - 1);
  m.low64 ^= swap64(m.high64);
  h128_t h = mult64to128(m.low64, P64_2);
  h.high64 += m.high64 * P64_2;
  h.low64 = xxh3_avalanche(h.low64);
  h.high64 = xxh3_avalanche(h.high64);
  return h;
}
static h128_t len_0to16(const uint8_t* in, size_t len, const uint8_t* sec, uint64_t seed) {
  if (len > 8) return len_9to16(in, len, sec, seed);
  if (len >= 4) return len_4to8(in, len, sec, seed);
  if (len) return len_1to3(in, len, sec, seed);
  h128_t h = {xxh64_avalanche(seed ^ (rd64(sec + 64) ^ rd64(sec + 72))),
              xxh64_avalanche(seed ^ (rd64(sec + 80) ^ rd64(sec + 88)))};
  return h;
}

/* ---- 17..240 ---- */
static inline uint64_t mix16B(const uint8_t* in, const uint8_t* sec, uint64_t seed) {
  return mul128_fold64(rd64(in) ^ (rd64(sec) + seed), rd64(in + 8) ^ (rd64(sec + 8) - seed));
}
static inline h128_t mix32B(h128_t acc, const uint8_t* in1, const uint8_t* in2, const uint8_t* sec, uint64_t seed) {
  acc.low64 += mix16B(in1, sec, seed);
  acc.low64 ^= rd64(in2) + rd64(in2 + 8);
  acc.high64 += mix16B(in2, sec + 16, seed);
  acc.high64 ^= rd64(in1) + rd64(in1 + 8);
  return acc;
}
static h128_t mid_finish(h128_t acc, size_t len, uint64_t seed) {
  h128_t h;
  h.low64 = acc.low64 + acc.high64;
  h.high64 = acc.low64 * P64_1 + acc.high64 * P64_4 + ((uint64_t)len - seed) * P64_2;
  h.low64 = xxh3_avalanche(h.low64);
  h.high64 = (uint64_t)0 - xxh3_avalanche(h.high64);
  return h;
}
static h128_t len_17to128(const uint8_t* in, size_t len, const uint8_t* sec, uint64_t seed) {
  h128_t acc = {(uint64_t)len * P64_1, 0};
  if (len > 32) {
    if (len > 64) {
      if (len > 96) acc = mix32B(acc, in + 48, in + len - 64, sec + 96, seed);
      acc = mix32B(acc, in + 32, in + len - 48, sec + 64, seed);
    }
    acc = mix32B(acc, in + 16, in + len - 32, sec + 32, seed);
  }
  acc = mix32B(acc, in, in + len - 16, sec, seed);
  return mid_finish(acc, len, seed);
}
static h128_t len_129to240(const uint8_t* in, size_t len, const uint8_t* sec, uint64_t seed) {
  h128_t acc = {(uint64_t)len * P64_1, 0};
  unsigned i;
  for (i = 32; i < 160; i += 32) acc = mix32B(acc, in + i - 32, in + i - 16, sec + i - 32, seed);
  acc.low64 = xxh3_avalanche(acc.low64);
  acc.high64 = xxh3_avalanche(acc.high64);
  for (i = 160; i <= len; i += 32)
    acc = mix32B(acc, in + i - 32, in + i - 16, sec + MIDSIZE_STARTOFFSET + i - 160, seed);
  acc = mix32B(acc, in + len - 16, in + len - 32, sec + SECRET_SIZE_MIN - MIDSIZE_LASTOFFSET - 16,
               (uint64_t)0 - seed);
  return mid_finish(acc, len, seed);
}

/* ---- > 240: stripes over the seed-derived secret ---- */
static void init_custom_secret(uint8_t* out, uint64_t seed) {
  for (int i = 0; i < SECRET_SIZE / 16; i++) {
    wr64(out + 16 * i, rd64(kSecret + 16 * i) + seed);
    wr64(out + 16 * i + 8, rd64(kSecret + 16 * i + 8) - seed);
  }
}
static inline void accumulate_512(uint64_t* acc, const uint8_t* in, const uint8_t* sec) {
  for (int l = 0; l < 8; l++) {
    uint64_t dv = rd64(in + 8 * l);
    uint64_t dk = dv ^ rd64(sec + 8 * l);
    acc[l ^ 1] += dv;
    acc[l] += (dk & 0xFFFFFFFFULL) * (dk >> 32);
  }
}
static inline void scramble(uint64_t* acc, const uint8_t* sec) {
  for (int l = 0; l < 8; l++) {
    uint64_t a = acc[l];
    a = xorshift64(a, 47);
    a ^= rd64(sec + 8 * l);
    a *= P32_1;
    acc[l] = a;
  }
}
static uint64_t merge_accs(const uint64_t* acc, const uint8_t* sec, uint64_t start) {
  uint64_t r = start;
  for (int i = 0; i < 4; i++)
    r += mul128_fold64(acc[2 * i] ^ rd64(sec + 16 * i), acc[2 * i + 1] ^ rd64(sec + 16 * i + 8));
  return xxh3_avalanche(r);
}
static h128_t hash_long(const uint8_t* in, size_t len, uint64_t seed) {
  uint8_t custom[SECRET_SIZE];
  const uint8_t* sec = kSecret;
  if (seed != 0) { init_custom_secret(custom, seed); sec = custom; }
  uint64_t acc[8] = {P32_3, P64_1, P64_2, P64_3, P64_4, P32_2, P64_5, P32_1};
  const size_t stripes_per_block = (SECRET_SIZE - STRIPE_LEN) / SECRET_CONSUME_RATE; /* 16 */
  const size_t block_len = STRIPE_LEN * stripes_per_block;                         /* 1024 */
  const size_t nb_blocks = (len - 1) / block_len;
  for (size_t n = 0; n < nb_blocks; n++) {
    for (size_t s = 0; s < stripes_per_block; s++)
      accumulate_512(acc, in + n * block_len + s * STRIPE_LEN, sec + s * SECRET_CONSUME_RATE);
    scramble(acc, sec + SECRET_SIZE - STRIPE_LEN);
  }
  const size_t nb_stripes = ((len - 1) - block_len * nb_blocks) / STRIPE_LEN;
  for (size_t s = 0; s < nb_stripes; s++)
    accumulate_512(acc, in + nb_blocks * block_len + s * STRIPE_LEN, sec + s * SECRET_CONSUME_RATE);
  accumulate_512(acc, in + len - STRIPE_LEN, sec + SECRET_SIZE - STRIPE_LEN - SECRET_LASTACC_START);
  h128_t h;
  h.low64 = merge_accs(acc, sec + SECRET_MERGEACCS_START, (uint64_t)len * P64_1);
  h.high64 = merge_accs(acc, sec + SECRET_SIZE - STRIPE_LEN - SECRET_MERGEACCS_START,
                        ~((uint64_t)len * P64_2));
  return h;
}

/* XXH3_128bits_withSeed; out16 = low64 LE || high64 LE (the XXH128_hash_t struct bytes). */
void oracle_xxh3_128_with_seed(const void* data, size_t len, uint64_t seed, uint8_t* out16) {
  const uint8_t* in = (const uint8_t*)data;
  h128_t h;
  if (len <= 16) h = len_0to16(in, len, kSecret, seed);
  else if (len <= 128) h = len_17to128(in, len, kSecret, seed);
  else if (len <= MIDSIZE_MAX) h = len_129to240(in, len, kSecret, seed);
  else h = hash_long(in, len, seed);
  wr64(out16, h.low64);
  wr64(out16 + 8, h.high64);
}

/* hash_util.cpp:18-45.  Returns 0, or -1 where the reference would CHECK-fail
 * (16 + 4*n >= 1024, hash_util.cpp:33).  prev16 and out16 may alias. */
int oracle_xxh3_128bits_hash(const uint8_t* prev16, const int32_t* tokens, size_t n_tokens,
                             uint32_t seed, uint8_t* out16) {
  if (prev16 == NULL) {
    oracle_xxh3_128_with_seed(tokens, sizeof(int32_t) * n_tokens, (uint64_t)seed, out16);
    return 0;
  }
  uint8_t key[1024];
  int32_t data_len = (int32_t)(sizeof(int32_t) * n_tokens + 16);
  if (!((int32_t)sizeof(key) > data_len)) return -1;
  memcpy(key, prev16, 16);
  memcpy(key + 16, tokens, sizeof(int32_t) * n_tokens);
  oracle_xxh3_128_with_seed(key, (size_t)data_len, (uint64_t)seed, out16);
  return 0;
}

/* The chain of global_kvcache_mgr.cpp:76-94 for one request: writes
 * floor(n_tokens/block_size) keys of 16 bytes.  Returns the number of keys, or
 * -1 on the reference's CHECK failure. */
long oracle_block_hash_chain(const int32_t* tokens, size_t n_tokens, uint32_t block_size,
                             uint32_t seed, uint8_t* keys_out) {
  if (block_size == 0) return -1;
  size_t nb = n_tokens / block_size;
  uint8_t key[16];
  for (size_t b = 0; b < nb; b++) {
    int rc = oracle_xxh3_128bits_hash(b == 0 ? NULL : key, tokens + b * block_size, block_size, seed, key);
    if (rc) return -1;
    memcpy(keys_out + 16 * b, key, 16);
  }
  return (long)nb;
}

/* Batch form over a CSR token layout (offsets in tokens; keys packed per request
 * at key_offsets[r]).  Used by the cpu_baseline leg. */
long oracle_block_hash_chain_batch(const int32_t* tokens, const int64_t* tok_offsets, size_t n_req,
                                   uint32_t block_size, uint32_t seed, uint8_t* keys_out,
                                   const int64_t* key_offsets) {
  long total = 0;
  for (size_t r = 0; r < n_req; r++) {
    long nb = oracle_block_hash_chain(tokens + tok_offsets[r], (size_t)(tok_offsets[r + 1] - tok_offsets[r]),
                                      block_size, seed, keys_out + 16 * key_offsets[r]);
    if (nb < 0) return -1;
    total += nb;
  }
  return total;
}
