/*
 * xllm_ingest.h — C-ABI of the H100 request-ingest + prefix-cache routing path.
 *
 * One shared library, libxllm_ingest.so (CUDA, sm_90a), replaces the CPU hot path
 * every request to an xllm-service front door traverses before PD dispatch:
 *
 *   Tokenizer::encode            xllm_service/tokenizer/tokenizer.h:32-33
 *                                (called at xllm_service/scheduler/scheduler.cpp:129)
 *   xxh3_128bits_hash            xllm_service/common/hash_util.h:56-58, hash_util.cpp:18-45
 *   GlobalKVCacheMgr::match      xllm_service/scheduler/managers/global_kvcache_mgr.h:39,
 *                                global_kvcache_mgr.cpp:73-131
 *   GlobalKVCacheMgr::record_updated_kvcaches / upload_kvcache
 *                                global_kvcache_mgr.cpp:177-247
 *   CacheAwareRouting::cost_function / select_instances_pair
 *                                xllm_service/scheduler/loadbalance_policy/cache_aware_routing.cpp:22-85
 *
 * Plain pointers and sizes only; no C++ or torch types.  Every entry point returns
 * 0 on success or a negative XLLM_ERR_* code and never aborts the process
 * (the reference's Rust shim panics, lib.rs:32,39,69,77,91; its C++ CHECKs abort).
 * xllm_last_error() returns a thread-local description of the last failure.
 *
 * Threading: a handle may be used from many threads; calls on one handle are
 * serialised internally (one CUDA stream per handle).  Create one handle per
 * worker thread / per GPU for concurrency (mirrors the reference's thread_local
 * tokenizer clone, scheduler.cpp:274-277) — handles created with
 * xllm_ingest_clone() share the device-resident tables.
 *
 * There is no CPU fallback inside this library: without a CUDA device every
 * compute entry point fails with XLLM_ERR_CUDA.
 */
#ifndef XLLM_INGEST_H_
#define XLLM_INGEST_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XLLM_OK 0
#define XLLM_ERR_INVALID_ARG (-1)
#define XLLM_ERR_CUDA (-2)
#define XLLM_ERR_IO (-3)
#define XLLM_ERR_FORMAT (-4)
#define XLLM_ERR_UNSUPPORTED (-5)
#define XLLM_ERR_CAPACITY (-6)
#define XLLM_ERR_NOMEM (-7)

#define XLLM_KEY_BYTES 16 /* sizeof(XXH128_hash_t), hash_util.h:14 */
#define XLLM_MAX_INSTANCES 64

typedef struct xllm_ingest* xllm_ingest_t;

/* Mirrors the hot-path gflags (xllm_service/common/global_gflags.cpp:60,114-118). */
typedef struct {
  const char* tokenizer_path; /* --tokenizer_path: directory holding tokenizer.model /
                                 tokenizer.json / a tiktoken vocab; NULL = no tokenizer */
  int32_t block_size;         /* --block_size, default 128 (0 => 128); must be in [1,251] (hash_util.cpp:29-33) */
  uint32_t xxh3_seed;         /* --xxh3_128bits_seed, default 1024 */
  int32_t device;             /* CUDA device ordinal */
  int32_t max_batch;          /* max requests per batch call (0 => 65536) */
  int64_t max_batch_bytes;    /* max total prompt bytes per batch call (0 => 64 MiB * ...; see DESIGN.md) */
  int32_t max_tokens;         /* max token ids per request (0 => 8192) */
  int64_t index_capacity;     /* max distinct block keys in the prefix index (0 => no index); with a sharded index:
                                 keys held by THIS GPU's shard */
  /* ---- hash-range-sharded prefix index over the GPUs of one box (all three zero / NULL => not sharded).  One
   * process per GPU; the GPU owning a block key is low64(key) >> (64 - log2(shard_world)); one NCCL all-to-all of
   * (hash128, request, block) tuples per batch and one of tier masks back (csrc/shard_exchange.cuh). */
  int32_t shard_world;        /* GPUs the index is split over: a power of two in [2, 32] (0 or 1 => not sharded) */
  int32_t shard_rank;         /* this process's rank in [0, shard_world); `device` above is its GPU */
  const void* nccl_unique_id; /* the 128 bytes xllm_shard_unique_id() produced on one rank, passed to every rank */
} xllm_ingest_config;

const char* xllm_last_error(void);
/* Rendezvous for a sharded index: call on ONE rank, hand the 128 bytes to all ranks (over whatever channel the
 * service already has: etcd, the launcher's env, torch.distributed in bench.py), then every rank calls
 * xllm_ingest_create with them — that call is collective (ncclCommInitRank).  NCCL is loaded with
 * dlopen("libnccl.so.2") on first use; XLLM_ERR_UNSUPPORTED when it is not installed. */
int xllm_shard_unique_id(void* out128);
/* Owner rank of a block key among `shard_world` GPUs (host-only helper: routing events, tests). */
int xllm_shard_owner(const uint8_t* key16, int32_t shard_world);
/* Device time of the last sharded match round on this handle, milliseconds: bucketing, exchange out, owner-side
 * probe, exchange back, first-miss scan + routing; and the tuples one message can carry / overflow repeats so far. */
typedef struct {
  float bucket_ms, exchange_out_ms, probe_ms, exchange_back_ms, score_ms;
  int64_t bucket_capacity;
  int64_t overflow_rounds;
} xllm_shard_stats;
int xllm_shard_last_stats(xllm_ingest_t h, xllm_shard_stats* out);
int xllm_ingest_create(const xllm_ingest_config* cfg, xllm_ingest_t* out);
int xllm_ingest_clone(xllm_ingest_t src, xllm_ingest_t* out);
void xllm_ingest_destroy(xllm_ingest_t h);

/* ---------------------------------------------------------------- block hash
 * Batch form of the chain in GlobalKVCacheMgr::match (global_kvcache_mgr.cpp:76-94):
 * request r owns tokens[tok_start[r] .. tok_start[r]+n_tok[r]) and gets
 * floor(n_tok[r]/block_size) keys of 16 bytes (low64 LE || high64 LE, the memcpy of
 * XXH128_hash_t at hash_util.cpp:26-27) written at keys + 16*key_start[r].
 * Trailing tokens past the last full block are ignored (global_kvcache_mgr.cpp:76).
 *
 * xllm_hash_blocks        : host pointers; copies in, runs the kernel, copies out.
 * xllm_hash_blocks_device : device pointers, asynchronous on `cuda_stream`
 *                           (a cudaStream_t passed as void*; NULL = the handle's stream).
 */
int xllm_hash_blocks(xllm_ingest_t h, int32_t n_req, const int32_t* tokens, int64_t n_tokens_total,
                     const int64_t* tok_start, const int32_t* n_tok, uint8_t* keys, int64_t n_keys_total,
                     const int64_t* key_start);
int xllm_hash_blocks_device(xllm_ingest_t h, int32_t n_req, const int32_t* d_tokens, const int64_t* d_tok_start,
                            const int32_t* d_n_tok, uint8_t* d_keys, const int64_t* d_key_start,
                            void* cuda_stream);

/* Single-call drop-in for xxh3_128bits_hash(pre_hash_value, token_ids, hash_value)
 * (hash_util.h:56-58): prev may be NULL (first block) and may alias out.  Fails with
 * XLLM_ERR_INVALID_ARG where the reference CHECK-fails (16 + 4*n >= 1024). */
int xllm_xxh3_128bits_hash(xllm_ingest_t h, const uint8_t* prev16, const int32_t* token_ids, size_t n_tokens,
                           uint8_t* out16);

/* ----------------------------------------------------------- prefix index (write side)
 * Instances are addressed by id 0..63 (bit positions of the per-tier instance masks that replace
 * CacheLocations' three unordered_set<string>, types.h:320-365); the host adaptor keeps name<->id.
 *
 * xllm_index_apply   = GlobalKVCacheMgr::record_updated_kvcaches(instance, KvCacheEvent)
 *                      (global_kvcache_mgr.cpp:177-225): keys are 16-byte XXH3Key values; stored,
 *                      then offload (HBM->DRAM, else DRAM->SSD), then removed; staged, NOT yet visible.
 * xllm_index_put / _erase = the replica path update_kvcache PUT / DELETE (:133-175); staged.
 * xllm_index_publish = upload_kvcache's local effect (:227-247): replays the staged events on the
 *                      device table (entries left empty are erased) and makes them visible to match.
 * With a sharded index every rank is given the same events; each keeps the keys it owns and ignores the rest
 * (xllm_index_get / _export / _size then report this rank's shard).
 */
int xllm_index_apply(xllm_ingest_t h, int32_t instance_id, const uint8_t* stored, size_t n_stored,
                     const uint8_t* offload, size_t n_offload, const uint8_t* removed, size_t n_removed);
int xllm_index_put(xllm_ingest_t h, const uint8_t* key16, uint64_t hbm_mask, uint64_t dram_mask, uint64_t ssd_mask);
int xllm_index_erase(xllm_ingest_t h, const uint8_t* key16);
/* Bulk xllm_index_put: what a replica or a restarted master does with the XLLM:CACHE:* pairs it lists from etcd
 * (global_kvcache_mgr.cpp:47-51 -> etcd_client.cpp:174-198); staged like the single form, publish afterwards. */
int xllm_index_put_bulk(xllm_ingest_t h, int64_t n, const uint8_t* keys /*[n][16]*/, const uint64_t* hbm_masks,
                        const uint64_t* dram_masks, const uint64_t* ssd_masks);
/* Snapshot of the published index: every live key with its three instance masks, in unspecified order — the
 * content the master holds in etcd under "XLLM:CACHE:" + key (etcd_client.cpp:122-137).  *n_keys = live keys;
 * returns XLLM_ERR_CAPACITY (with *n_keys set, the first `capacity` rows filled) when capacity is too small.
 * host/index_wire.h turns rows into / from the reference's etcd keys and CacheLocations JSON (types.h:320-365). */
int xllm_index_export(xllm_ingest_t h, int64_t capacity, uint8_t* keys /*[capacity][16]*/, uint64_t* hbm_masks,
                      uint64_t* dram_masks, uint64_t* ssd_masks, int64_t* n_keys);
int xllm_index_publish(xllm_ingest_t h);
/* An instance left the cluster (InstanceMgr::deregister_instance): clears its bit in every entry of the published
 * index at once — the sum of the removed_cache events the reference would need for each of its blocks — erasing
 * entries left empty, so the id can be handed to a new instance.  Staged events are not touched. */
int xllm_index_clear_instance(xllm_ingest_t h, int32_t instance_id);
/* Table health as of the last publish: live keys, tombstones (erased slots not yet reclaimed) and how many times the
 * table was rebuilt in place (publish does that when live + tombstones exceed 70 % of the slots). */
int xllm_index_stats(xllm_ingest_t h, int64_t* live_keys, int64_t* tombstones, int64_t* rebuilds);
int xllm_index_size(xllm_ingest_t h, int64_t* n_keys);
int xllm_index_get(xllm_ingest_t h, const uint8_t* key16, uint64_t masks3[3], int32_t* found);

/* Instance view read by the routing step: InstanceMgr's instances_ / load_metrics_ as consumed by
 * get_load_metrics (instance_mgr.cpp:287-359).  type: 0 DEFAULT, 1 PREFILL, 2 DECODE, 3 MIX. */
int xllm_set_instance(xllm_ingest_t h, int32_t instance_id, int32_t type, int32_t schedulable);
int xllm_set_load_metrics(xllm_ingest_t h, int32_t instance_id, int32_t has_metrics, uint64_t waiting_requests_num,
                          float gpu_cache_usage_perc);

/* ------------------------------------------------------------- match + cache-aware routing
 * xllm_match_out = OverlapScores (types.h:376-403) with instance ids for names; a score of 0 means the
 * instance is absent from that score map.  xllm_routing_out = Routing (types.h:43-55) + the return
 * value of CacheAwareRouting::select_instances_pair (ok == 0 <=> false, "No node available").
 * Ties in cost_function are broken by the lowest instance id (the reference: unordered_map order).
 */
typedef struct {
  uint32_t max_block_num;
  uint32_t max_matched_block_num;
  uint64_t instances;
  uint16_t hbm_instance_score[XLLM_MAX_INSTANCES];
  uint16_t dram_instance_score[XLLM_MAX_INSTANCES];
  uint16_t ssd_instance_score[XLLM_MAX_INSTANCES];
} xllm_match_out;
typedef struct {
  int32_t prefill_id; /* -1: prefill_name left empty */
  int32_t decode_id;
  int32_t ok;
  float prefill_score;
  float decode_score;
} xllm_routing_out;

/* keys: the block keys of all requests; request r owns n_blocks[r] keys starting at key_start[r].
 * match / routing may be NULL.  Host-pointer and device-pointer forms.
 * n_blocks[r] must be at most 65 535 (the scores are 16-bit).  xllm_match_route checks it and fails with
 * XLLM_ERR_INVALID_ARG; xllm_match_route_device and xllm_score_route_device read n_blocks on the device and cannot
 * check it without a synchronisation, so there the limit is the caller's to keep.
 * The device-pointer calls of one handle share its counters and scratch: issue them in order on one stream.
 * With a sharded index these two calls and xllm_ingest_batch (when match / routing is requested) are COLLECTIVE: every
 * rank must make the call once per batch (each with its own requests, n_req may be 0); they synchronise the stream. */
int xllm_match_route(xllm_ingest_t h, int32_t n_req, const uint8_t* keys, int64_t n_keys_total,
                     const int64_t* key_start, const int32_t* n_blocks, xllm_match_out* match,
                     xllm_routing_out* routing);
int xllm_match_route_device(xllm_ingest_t h, int32_t n_req, const uint8_t* d_keys, int64_t n_keys_total,
                            const int64_t* d_key_start, const int32_t* d_n_blocks, xllm_match_out* d_match,
                            xllm_routing_out* d_routing, void* cuda_stream);
/* The two halves, for a hash-range-sharded index (keys exchanged between GPUs in between):
 * probe: masks3[k] = {hbm, dram, ssd} of keys[k] (zeros when absent); score: first-miss scan + routing. */
int xllm_index_probe_device(xllm_ingest_t h, const uint8_t* d_keys, int64_t n_keys, uint64_t* d_masks3,
                            void* cuda_stream);
int xllm_score_route_device(xllm_ingest_t h, int32_t n_req, const uint64_t* d_masks3, const int64_t* d_key_start,
                            const int32_t* d_n_blocks, xllm_match_out* d_match, xllm_routing_out* d_routing,
                            void* cuda_stream);

/* ------------------------------------------------------------------ tokenize
 * Batch form of Tokenizer::encode (xllm_service/tokenizer/tokenizer.h:32-33; the service calls
 * it once per request at scheduler.cpp:129).  text holds all prompts back to back;
 * offsets[n_req + 1] are byte offsets.  Request r's ids are written to ids + r*ids_stride
 * (at most ids_stride of them); n_ids[r] is the full count; status[r] is 0 (ok),
 * XLLM_ENC_TRUNCATED (count > ids_stride: call again with a larger stride),
 * XLLM_ERR_CAPACITY (a single pre-token longer than the device scratch holds) or, on the HF backend,
 * XLLM_ERR_INVALID_ARG (malformed UTF-8: the reference's Rust shim panics there, lib.rs:91) or
 * XLLM_ERR_UNSUPPORTED (tokenizer.json with normalizer NFC and a text that is not provably in NFC already).
 * An empty prompt yields 0 ids (sentencepiece_tokenizer.cpp:117-120) plus, on the HF backend, the
 * template's special tokens.
 * Backend, in the order of TokenizerFactory::create_tokenizer (tokenizer_factory.cpp:9-32):
 * `<tokenizer_path>/tokenizer.json` -> HF byte-level BPE (fast_tokenizer.cpp:8-30); tokenizer_config.json with
 * tokenizer_class TikTokenTokenizer -> tiktoken (tiktoken_tokenizer.cpp:115-294); else SentencePiece (BPE or
 * Unigram) `<tokenizer_path>/tokenizer.model` (sentencepiece_tokenizer.cpp:47-50).  A model outside the supported
 * envelope fails xllm_ingest_create with XLLM_ERR_UNSUPPORTED; a handle without a tokenizer returns it here.
 */
#define XLLM_ENC_TRUNCATED 1
int xllm_encode_batch(xllm_ingest_t h, int32_t n_req, const uint8_t* text, const int64_t* offsets, int32_t* ids,
                      int64_t ids_stride, int32_t* n_ids, int32_t* status);
/* Diagnostics: xllm_encode_batch without the id download, plus how long every warp of the tokenizer's persistent
 * grid (one warp takes one request at a time from a shared counter) stayed busy, in nanoseconds; *n_warps = warps
 * launched (the first min(n_warps, warp_cap) entries of warp_ns are filled).  max / mean of those numbers is the
 * length tail a variable-length batch leaves at the end of the kernel. */
int xllm_encode_batch_profile(xllm_ingest_t h, int32_t n_req, const uint8_t* text, const int64_t* offsets,
                              int64_t ids_stride, int32_t* n_ids, int32_t* status, uint64_t* warp_ns, int32_t warp_cap,
                              int32_t* n_warps);
int xllm_encode_batch_device(xllm_ingest_t h, int32_t n_req, const uint8_t* d_text, const int64_t* d_offsets,
                             int32_t* d_ids, int64_t ids_stride, int32_t* d_n_ids, int32_t* d_status,
                             void* cuda_stream);
/* ------------------------------------------------------------ the whole path, one call
 * What Scheduler::schedule does per request between scheduler.cpp:128 and :135 — Tokenizer::encode,
 * then CacheAwareRouting::select_instances_pair (GlobalKVCacheMgr::match + cost_function) — for a
 * whole batch: host text in, token ids / block keys / OverlapScores / Routing out.  The batch is
 * pipelined in chunks over several CUDA streams; pass page-locked buffers (xllm_host_alloc) so
 * the PCIe copies overlap the kernels.  keys / match / routing may be NULL to skip those outputs
 * (match or routing != NULL requires an index).  keys_stride = 16-byte keys per request row
 * (0 => ids_stride / block_size); rows are zero-padded past floor(n_ids/block_size).  keys_stride also caps the
 * blocks that are hashed and matched: a row's keys, match and routing cover its first
 * min(keys_stride, floor(min(n_ids, ids_stride)/block_size)) blocks.
 * Match scores are 16-bit (xllm_match_out): with match or routing requested, a batch whose rows can hold more than
 * 65 535 blocks (min(keys_stride, ids_stride / block_size) > 65 535) is refused with XLLM_ERR_INVALID_ARG before any
 * work is queued.  Keys alone have no such limit.
 */
typedef struct {
  int32_t n_req;
  const uint8_t* text;    /* all prompts back to back */
  const int64_t* offsets; /* [n_req + 1] byte offsets into text */
  int32_t* ids;           /* [n_req][ids_stride] */
  int64_t ids_stride;
  int32_t* n_ids;         /* [n_req] full token counts */
  int32_t* status;        /* [n_req] 0 / XLLM_ENC_TRUNCATED / XLLM_ERR_CAPACITY / _INVALID_ARG / _UNSUPPORTED */
  uint8_t* keys;          /* [n_req][keys_stride][16] or NULL */
  int64_t keys_stride;
  xllm_match_out* match;     /* [n_req] or NULL */
  xllm_routing_out* routing; /* [n_req] or NULL */
  /* Opt-in narrow download: when non-NULL the token ids are delivered HERE as uint16 rows [n_req][ids_stride] and
   * `ids` is not written (it may be NULL).  Only for vocabularies below 65 536 pieces (XLLM_ERR_UNSUPPORTED
   * otherwise).  Token ids are half of the bytes that cross PCIe on the way back; a caller that copies them into its
   * own std::vector<int32_t> anyway (Request::token_ids — host/ingest_batcher.h does) widens during that copy. */
  uint16_t* ids_u16;
} xllm_ingest_io;
int xllm_ingest_batch(xllm_ingest_t h, const xllm_ingest_io* io);

/* ---------------------------------------------- requests made of text pieces AND ready-made token ids (config 5)
 * A multimodal request reaches the scheduler as text interleaved with spans that are already token ids — runs of
 * image-placeholder ids expanded by the front end (the reference only carries a "mm place holder" string through the
 * chat template, jinja_chat_template.cpp:119-137, and appends whatever Tokenizer::encode returns to
 * Request::token_ids, scheduler.cpp:128-132, sentencepiece_tokenizer.cpp:122-126).  This entry point keeps that
 * append semantics: a request is a list of segments; a text segment is tokenised exactly like one
 * Tokenizer::encode call on that piece (own dummy prefix / whitespace rules / template ids), an id segment is copied
 * verbatim; the request's token ids are the concatenation, and block keys / match / routing are computed over it as
 * usual — the id spans bypass BPE but are hashed and matched.
 *   io->text / io->offsets describe the TEXT PIECES of all requests back to back, in request order
 *   (offsets[n_pieces + 1]); every other field of io keeps its per-request meaning (n_req, ids rows, n_ids, ...).
 *   seg_len[s] >= 0: an id segment of that many ids, taken in order from span_ids; seg_len[s] == -1: the next text
 *   piece.  status[r]: the first failing piece's error, else XLLM_ENC_TRUNCATED / 0. */
typedef struct {
  int64_t n_segments;           /* segments of all requests */
  const int32_t* req_seg_start; /* [n_req + 1]: request r owns segments [req_seg_start[r], req_seg_start[r + 1]) */
  const int32_t* seg_len;       /* [n_segments] */
  const int32_t* span_ids;      /* [n_span_ids] all ready-made ids back to back, in segment order */
  int64_t n_span_ids;
} xllm_segments;
int xllm_ingest_batch_segments(xllm_ingest_t h, const xllm_ingest_io* io, const xllm_segments* seg);
/* Pipeline chunking of xllm_ingest_batch: at most chunk_requests requests and chunk_bytes text bytes
 * per chunk (defaults 4096 / 96 MiB; chunk sizes ramp up from chunk_requests/16 and taper off at the end;
 * 4 chunks in flight over one upload, one kernel and one download stream). */
int xllm_set_pipeline(xllm_ingest_t h, int32_t chunk_requests, int64_t chunk_bytes);
/* Word memo of the tokenizer kernels (word bytes -> token ids, immutable entries, one table per launch site).
 * persist_requests == 0 (default): every encode launch starts from an empty table, nothing is carried from one batch
 * to the next.  persist_requests == N > 0: a table is kept across launches and cleared once it has seen N requests —
 * the service setting (host/ingest_batcher.h): small batches no longer pay for the cold table, results are identical
 * either way (a stale table is only ever less complete).  Env XLLM_SP_MEMO_PERSIST=N sets it at create. */
int xllm_set_memo_policy(xllm_ingest_t h, int64_t persist_requests);
/* Chunks and kernel launches of the most recent xllm_ingest_batch on this handle (for launch accounting). */
int xllm_last_batch_stats(xllm_ingest_t h, int32_t* n_chunks, int32_t* n_kernel_launches);
/* Page-locked host memory for the batch buffers. */
int xllm_host_alloc(void** out, size_t bytes);
void xllm_host_free(void* p);

/* Host-only: parse a tokenizer directory and report the tables the device encoder would use
 * (no CUDA needed).  split_mode: 1 = words split before every U+2581, 2 = before a U+2581 not
 * preceded by U+2581, 0 = the vocabulary allows no exact pre-split. */
typedef struct {
  int32_t n_pieces;
  int32_t n_symbols;      /* pieces + single chars that only occur inside pieces */
  int32_t n_pair_slots;   /* open-addressing slots of the (left,right)->(priority,merged) table */
  int32_t n_pairs;        /* occupied slots */
  int32_t split_mode;
  int32_t max_unit_out;   /* longest normalizer replacement after whitespace escaping (bytes) */
  int32_t byte_fallback;
  int32_t unk_id;
  int32_t trie_units;
  int32_t avg_probe_x100; /* mean probes per successful pair lookup, x100 */
  int32_t max_probe;      /* longest probe chain of a stored pair */
} xllm_tokenizer_info;
int xllm_tokenizer_probe(const char* tokenizer_path, xllm_tokenizer_info* out);

/* Vocabulary size = GetPieceSize() (sentencepiece_tokenizer.cpp:251). */
int xllm_vocab_size(xllm_ingest_t h, int32_t* out);

#ifdef __cplusplus
}
#endif
#endif /* XLLM_INGEST_H_ */
