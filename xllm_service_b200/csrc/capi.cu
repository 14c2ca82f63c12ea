// capi.cu — the extern "C" boundary declared in include/xllm_ingest.h.
#include <stdarg.h>
#include <string.h>

#include <new>

#include "../../include/xllm_ingest.h"
#include "handle.h"

namespace xllm {

uint32_t sp_pair_slot_fwd(uint32_t a, uint32_t b, uint32_t n_slots);  // sp_model.cc

static thread_local char g_last_error[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

int DevBuf::reserve(size_t bytes) {
  if (bytes <= cap) return XLLM_OK;
  release();
  size_t want = bytes + bytes / 4 + 256;
  cudaError_t e = cudaMalloc(&p, want);
  if (e != cudaSuccess) {
    p = nullptr;
    cap = 0;
    set_last_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    return XLLM_ERR_NOMEM;
  }
  cap = want;
  return XLLM_OK;
}
void DevBuf::release() {
  if (p) cudaFree(p);
  p = nullptr;
  cap = 0;
}
int PinBuf::reserve(size_t bytes) {
  if (bytes <= cap) return XLLM_OK;
  release();
  size_t want = bytes + bytes / 4 + 256;
  cudaError_t e = cudaMallocHost(&p, want);
  if (e != cudaSuccess) {
    p = nullptr;
    cap = 0;
    set_last_error("cudaMallocHost(%zu) failed: %s", want, cudaGetErrorString(e));
    return XLLM_ERR_NOMEM;
  }
  cap = want;
  return XLLM_OK;
}
void PinBuf::release() {
  if (p) cudaFreeHost(p);
  p = nullptr;
  cap = 0;
}

int encode_reserve(xllm_ingest* h, int n_req, DevBuf* scratch, DevBuf* memo_buf, int64_t* memo_age, SpMemo* memo,
                   SpEncodePlan* plan) {
  XLLM_CUDA_TRY(sp_encode_plan(h->sp_dev->dev(), n_req, h->memo_slots != 0, h->sp_warm, plan,
                               h->nfc_policy == XLLM_NFC_VERIFY));
  XLLM_TRY_RC(scratch->reserve(plan->scratch_bytes));
  *memo = SpMemo();
  if (plan->memo) {
    XLLM_TRY_RC(memo_buf->reserve((size_t)h->memo_slots * 32));
    memo->table = memo_buf->p;
    memo->slots = h->memo_slots;
    memo->clear = memo_needs_clear(h->memo_persist_requests, memo_age, n_req);
  }
  if (plan->warm) {   // one arena per handle: its launches, pipeline chunks included, run one after the other
    XLLM_TRY_RC(h->d_arena.reserve(plan->arena_bytes));   // the full grid's worth: never regrown
    memo->warm = true;
    memo->arena = h->d_arena.p;
    memo->arena_bytes = plan->arena_bytes;
  }
  return XLLM_OK;
}

}  // namespace xllm

using namespace xllm;

extern "C" {

const char* xllm_last_error(void) { return g_last_error; }

int xllm_ingest_create(const xllm_ingest_config* cfg, xllm_ingest_t* out) {
  if (!cfg || !out) {
    set_last_error("xllm_ingest_create: null argument");
    return XLLM_ERR_INVALID_ARG;
  }
  *out = nullptr;
  const int bs = cfg->block_size == 0 ? 128 : cfg->block_size;
  // hash_util.cpp:29-33: CHECK_GT(1024, 4*block_size + 16)
  if (bs < 1 || 4 * bs + 16 >= 1024) {
    set_last_error("block_size %d outside [1,251] (hash_util.cpp:29-33 frame limit)", bs);
    return XLLM_ERR_INVALID_ARG;
  }
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0) {
    set_last_error("no CUDA device: %s (this library has no CPU fallback)", cudaGetErrorString(e));
    return XLLM_ERR_CUDA;
  }
  if (cfg->device < 0 || cfg->device >= n_dev) {
    set_last_error("device %d out of range [0,%d)", cfg->device, n_dev);
    return XLLM_ERR_INVALID_ARG;
  }
  xllm_ingest* h = new (std::nothrow) xllm_ingest();
  if (!h) return XLLM_ERR_NOMEM;
  h->device = cfg->device;
  h->block_size = bs;
  h->seed = cfg->xxh3_seed;
  h->max_batch = cfg->max_batch > 0 ? cfg->max_batch : 65536;
  h->max_tokens = cfg->max_tokens > 0 ? cfg->max_tokens : 8192;
  xxh3_make_consts(h->seed, &h->xxh);
  if (cudaSetDevice(h->device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMalloc(&h->d_task_counter, 64) != cudaSuccess) {
    set_last_error("CUDA initialisation failed on device %d: %s", h->device,
                   cudaGetErrorString(cudaGetLastError()));
    xllm_ingest_destroy(h);
    return XLLM_ERR_CUDA;
  }
  if (cfg->tokenizer_path && cfg->tokenizer_path[0]) {
    h->tokenizer_path = cfg->tokenizer_path;
    h->sp_tables = std::make_shared<SpTables>();
    int rc = load_tokenizer_tables(h->tokenizer_path, h->sp_tables.get());
    if (rc != XLLM_OK) {
      set_last_error("tokenizer %s: %s", cfg->tokenizer_path, h->sp_tables->error.c_str());
      xllm_ingest_destroy(h);
      return rc;
    }
    h->memo_slots = sp_memo_default_slots();
    if (const char* w = getenv("XLLM_SP_MEMO_PERSIST")) h->memo_persist_requests = atoll(w) > 0 ? atoll(w) : 0;
    if (const char* w = getenv("XLLM_SP_WARM")) h->sp_warm = atoi(w) != 0;
    if (const char* w = getenv("XLLM_HF_NFC_VERIFY")) h->nfc_policy = atoi(w) != 0 ? XLLM_NFC_VERIFY : XLLM_NFC_PROVE_INERT;
    if (const char* w = getenv("XLLM_PIPE_SLOTS")) {
      const int v = atoi(w);
      if (v >= 1 && v <= kPipeSlots) h->pipe_slots = v;
    }
    h->sp_dev = std::make_shared<SpDeviceModel>();
    rc = h->sp_dev->upload(*h->sp_tables);
    if (rc != XLLM_OK) {
      xllm_ingest_destroy(h);
      return rc;
    }
  }
  h->inst_host = std::make_shared<InstanceTable>();
  memset(h->inst_host.get(), 0, sizeof(InstanceTable));
  h->index_mu = std::make_shared<std::mutex>();
  if (cudaMalloc(&h->d_inst, sizeof(InstanceTable)) != cudaSuccess) {
    set_last_error("cudaMalloc(InstanceTable) failed");
    xllm_ingest_destroy(h);
    return XLLM_ERR_NOMEM;
  }
  if (cfg->index_capacity > 0) {
    h->index = std::make_shared<PrefixIndex>();
    int rc = h->index->init(cfg->index_capacity);
    if (rc != XLLM_OK) {
      xllm_ingest_destroy(h);
      return rc;
    }
    h->index_read_ev = h->index->register_reader();
  }
  if (cfg->shard_world > 1) {
    if (!h->index) {
      set_last_error("a sharded index needs index_capacity > 0 (keys held by this GPU's shard)");
      xllm_ingest_destroy(h);
      return XLLM_ERR_INVALID_ARG;
    }
    // tuples one message can carry: 1.5x the mean bucket of the largest batch the config describes.  Every rank
    // passes the same config, so every rank derives the same capacity (shard_exchange.cuh).
    const int64_t blocks = (h->max_tokens + bs - 1) / bs;
    const int64_t cap = (int64_t)h->max_batch * blocks * 3 / (2 * (int64_t)cfg->shard_world) + 1024;
    h->shard = std::make_shared<ShardExchange>();
    const int rc = h->shard->init(cfg->shard_world, cfg->shard_rank, cfg->nccl_unique_id, h->device, cap);
    if (rc != XLLM_OK) {
      xllm_ingest_destroy(h);
      return rc;
    }
  }
  *out = h;
  return XLLM_OK;
}

int xllm_ingest_clone(xllm_ingest_t src, xllm_ingest_t* out) {
  if (!src || !out) {
    set_last_error("xllm_ingest_clone: null argument");
    return XLLM_ERR_INVALID_ARG;
  }
  xllm_ingest_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.block_size = src->block_size;
  cfg.xxh3_seed = src->seed;
  cfg.device = src->device;
  cfg.max_batch = src->max_batch;
  cfg.max_tokens = src->max_tokens;
  int rc = xllm_ingest_create(&cfg, out);
  if (rc != XLLM_OK) return rc;
  // clones share the device-resident tokenizer tables (the reference reloads the model per clone:
  // sentencepiece_tokenizer.cpp:254-256)
  (*out)->sp_tables = src->sp_tables;
  (*out)->sp_dev = src->sp_dev;
  (*out)->memo_slots = src->memo_slots;
  (*out)->memo_persist_requests = src->memo_persist_requests;
  (*out)->nfc_policy = src->nfc_policy;
  (*out)->sp_warm = src->sp_warm;
  (*out)->pipe_slots = src->pipe_slots;
  (*out)->tokenizer_path = src->tokenizer_path;
  (*out)->shard = src->shard;
  (*out)->index = src->index;
  if (src->index) (*out)->index_read_ev = src->index->register_reader();
  (*out)->index_mu = src->index_mu;
  (*out)->inst_host = src->inst_host;
  return XLLM_OK;
}

void xllm_ingest_destroy(xllm_ingest_t h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (int k = 0; k < 3; ++k)
    if (h->pipe_stream[k]) cudaStreamSynchronize(h->pipe_stream[k]);
  if (h->index && h->index_read_ev) h->index->unregister_reader(h->index_read_ev);
  h->index_read_ev = nullptr;
  h->d_tokens.release();
  h->d_tok_start.release();
  h->d_n_tok.release();
  h->d_keys.release();
  h->d_key_start.release();
  h->d_text.release();
  h->d_offsets.release();
  h->d_ids.release();
  h->d_n_ids.release();
  h->d_status.release();
  h->d_defer.release();
  h->d_memo.release();
  h->d_arena.release();
  h->d_masks.release();
  h->d_match.release();
  h->d_routing.release();
  h->d_nblk.release();
  h->d_all_keys.release();
  h->d_all_key_start.release();
  h->d_all_n_blocks.release();
  h->d_all_match.release();
  h->d_all_routing.release();
  if (h->d_inst) cudaFree(h->d_inst);
  for (int i = 0; i < kPipeSlots; ++i) h->pipe[i].release();
  for (int k = 0; k < 3; ++k)
    if (h->pipe_stream[k]) cudaStreamDestroy(h->pipe_stream[k]);
  if (h->d_task_counter) cudaFree(h->d_task_counter);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

int xllm_hash_blocks_device(xllm_ingest_t h, int32_t n_req, const int32_t* d_tokens, const int64_t* d_tok_start,
                            const int32_t* d_n_tok, uint8_t* d_keys, const int64_t* d_key_start,
                            void* cuda_stream) {
  if (!h || n_req < 0 || (n_req > 0 && (!d_tokens || !d_tok_start || !d_n_tok || !d_keys || !d_key_start))) {
    set_last_error("xllm_hash_blocks_device: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  if (n_req == 0) return XLLM_OK;
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : h->stream;
  XLLM_CUDA_TRY(xxh3_chain_launch(d_tokens, d_tok_start, d_n_tok, d_keys, d_key_start, n_req, h->block_size, h->xxh,
                                  h->d_task_counter, s));
  return XLLM_OK;
}

int xllm_hash_blocks(xllm_ingest_t h, int32_t n_req, const int32_t* tokens, int64_t n_tokens_total,
                     const int64_t* tok_start, const int32_t* n_tok, uint8_t* keys, int64_t n_keys_total,
                     const int64_t* key_start) {
  if (!h || n_req < 0 || n_tokens_total < 0 || n_keys_total < 0 ||
      (n_req > 0 && (!tok_start || !n_tok || !key_start)) || (n_tokens_total > 0 && !tokens) ||
      (n_keys_total > 0 && !keys)) {
    set_last_error("xllm_hash_blocks: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  if (n_req == 0) return XLLM_OK;
  // bounds: every row must lie inside the buffers the caller described
  for (int32_t r = 0; r < n_req; ++r) {
    const int64_t nb = n_tok[r] < 0 ? -1 : n_tok[r] / h->block_size;
    if (nb < 0 || tok_start[r] < 0 || tok_start[r] + n_tok[r] > n_tokens_total || key_start[r] < 0 ||
        key_start[r] + nb > n_keys_total) {
      set_last_error("xllm_hash_blocks: request %d out of bounds", r);
      return XLLM_ERR_INVALID_ARG;
    }
  }
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  XLLM_TRY_RC(h->d_tokens.reserve((size_t)n_tokens_total * 4 + 16));
  XLLM_TRY_RC(h->d_tok_start.reserve((size_t)n_req * 8));
  XLLM_TRY_RC(h->d_n_tok.reserve((size_t)n_req * 4));
  XLLM_TRY_RC(h->d_keys.reserve((size_t)n_keys_total * 16 + 16));
  XLLM_TRY_RC(h->d_key_start.reserve((size_t)n_req * 8));
  cudaStream_t s = h->stream;
  XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_tokens.p, tokens, (size_t)n_tokens_total * 4, cudaMemcpyHostToDevice, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_tok_start.p, tok_start, (size_t)n_req * 8, cudaMemcpyHostToDevice, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_n_tok.p, n_tok, (size_t)n_req * 4, cudaMemcpyHostToDevice, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_key_start.p, key_start, (size_t)n_req * 8, cudaMemcpyHostToDevice, s));
  XLLM_CUDA_TRY(xxh3_chain_launch(h->d_tokens.as<int32_t>(), h->d_tok_start.as<int64_t>(), h->d_n_tok.as<int32_t>(),
                                  h->d_keys.as<uint8_t>(), h->d_key_start.as<int64_t>(), n_req, h->block_size,
                                  h->xxh, h->d_task_counter, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(keys, h->d_keys.p, (size_t)n_keys_total * 16, cudaMemcpyDeviceToHost, s));
  XLLM_CUDA_TRY(cudaStreamSynchronize(s));
  return XLLM_OK;
}

int xllm_xxh3_128bits_hash(xllm_ingest_t h, const uint8_t* prev16, const int32_t* token_ids, size_t n_tokens,
                           uint8_t* out16) {
  if (!h || !out16 || (n_tokens > 0 && !token_ids)) {
    set_last_error("xllm_xxh3_128bits_hash: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  // hash_util.cpp:31-33
  if (prev16 && !(1024 > (int64_t)(4 * n_tokens + 16))) {
    set_last_error("key size is too small (hash_util.cpp:33): %zu tokens", n_tokens);
    return XLLM_ERR_INVALID_ARG;
  }
  if (n_tokens > 100000000) return XLLM_ERR_INVALID_ARG;
  // One (possibly chained) hash = the generic kernel over a frame of int32 "tokens".
  // A chained call hashes prev16 || tokens, i.e. an unchained hash of 4 + n tokens.
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  const size_t n = n_tokens + (prev16 ? 4 : 0);
  XLLM_TRY_RC(h->d_tokens.reserve(n * 4 + 16));
  XLLM_TRY_RC(h->d_keys.reserve(32));
  cudaStream_t s = h->stream;
  uint8_t* dt = h->d_tokens.as<uint8_t>();
  if (prev16) XLLM_CUDA_TRY(cudaMemcpyAsync(dt, prev16, 16, cudaMemcpyHostToDevice, s));
  if (n_tokens)
    XLLM_CUDA_TRY(cudaMemcpyAsync(dt + (prev16 ? 16 : 0), token_ids, n_tokens * 4, cudaMemcpyHostToDevice, s));
  XLLM_CUDA_TRY(xxh3_single_launch(h->d_tokens.as<uint8_t>(), n * 4, h->d_keys.as<uint8_t>(), h->xxh, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(out16, h->d_keys.p, 16, cudaMemcpyDeviceToHost, s));
  XLLM_CUDA_TRY(cudaStreamSynchronize(s));
  return XLLM_OK;
}

// ------------------------------------------------------------------ prefix index
static inline bool owns_key(xllm_ingest_t h, const uint8_t* key16) {
  if (!h->shard) return true;
  uint64_t lo;
  memcpy(&lo, key16, 8);
  return h->shard->owns(lo);
}
int xllm_shard_unique_id(void* out128) {
  if (!out128) return XLLM_ERR_INVALID_ARG;
  return ShardExchange::unique_id(out128);
}
int xllm_shard_owner(const uint8_t* key16, int32_t shard_world) {
  if (!key16 || shard_world < 1 || (shard_world & (shard_world - 1)) != 0) return XLLM_ERR_INVALID_ARG;
  int l2 = 0;
  while ((1 << l2) < shard_world) ++l2;
  uint64_t lo;
  memcpy(&lo, key16, 8);
  return shard_owner_of(lo, l2);
}
int xllm_shard_last_stats(xllm_ingest_t h, xllm_shard_stats* out) {
  if (!h || !out) return XLLM_ERR_INVALID_ARG;
  if (!h->shard) {
    set_last_error("this handle's index is not sharded");
    return XLLM_ERR_UNSUPPORTED;
  }
  const ShardTimes& t = h->shard->last_times();
  out->bucket_ms = t.bucket_ms;
  out->exchange_out_ms = t.exchange_out_ms;
  out->probe_ms = t.probe_ms;
  out->exchange_back_ms = t.exchange_back_ms;
  out->score_ms = t.score_ms;
  out->bucket_capacity = h->shard->bucket_capacity();
  out->overflow_rounds = h->shard->overflow_rounds();
  return XLLM_OK;
}
static int need_index(xllm_ingest_t h) {
  if (!h) {
    set_last_error("null handle");
    return XLLM_ERR_INVALID_ARG;
  }
  if (!h->index || !h->index->ready()) {
    set_last_error("prefix index not configured (index_capacity == 0)");
    return XLLM_ERR_UNSUPPORTED;
  }
  return XLLM_OK;
}

int xllm_index_apply(xllm_ingest_t h, int32_t instance_id, const uint8_t* stored, size_t n_stored,
                     const uint8_t* offload, size_t n_offload, const uint8_t* removed, size_t n_removed) {
  XLLM_TRY_RC(need_index(h));
  if (instance_id < 0 || instance_id >= kMaxInstances || (n_stored && !stored) || (n_offload && !offload) ||
      (n_removed && !removed)) {
    set_last_error("xllm_index_apply: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  std::lock_guard<std::mutex> lock(*h->index_mu);
  if (h->shard) {   // this rank keeps the keys of its own hash range
    std::vector<uint8_t> mine[3];
    const uint8_t* src[3] = {stored, offload, removed};
    const size_t cnt[3] = {n_stored, n_offload, n_removed};
    for (int t = 0; t < 3; ++t)
      for (size_t i = 0; i < cnt[t]; ++i)
        if (owns_key(h, src[t] + 16 * i)) mine[t].insert(mine[t].end(), src[t] + 16 * i, src[t] + 16 * i + 16);
    h->index->record(instance_id, mine[0].data(), mine[0].size() / 16, mine[1].data(), mine[1].size() / 16,
                     mine[2].data(), mine[2].size() / 16);
    return XLLM_OK;
  }
  h->index->record(instance_id, stored, n_stored, offload, n_offload, removed, n_removed);
  return XLLM_OK;
}
int xllm_index_put(xllm_ingest_t h, const uint8_t* key16, uint64_t hbm, uint64_t dram, uint64_t ssd) {
  XLLM_TRY_RC(need_index(h));
  if (!key16) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(*h->index_mu);
  if (!owns_key(h, key16)) return XLLM_OK;
  h->index->put(key16, hbm, dram, ssd);
  return XLLM_OK;
}
int xllm_index_put_bulk(xllm_ingest_t h, int64_t n, const uint8_t* keys, const uint64_t* hbm, const uint64_t* dram,
                        const uint64_t* ssd) {
  XLLM_TRY_RC(need_index(h));
  if (n < 0 || (n > 0 && (!keys || !hbm || !dram || !ssd))) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(*h->index_mu);
  for (int64_t i = 0; i < n; ++i)
    if (owns_key(h, keys + 16 * i)) h->index->put(keys + 16 * i, hbm[i], dram[i], ssd[i]);
  return XLLM_OK;
}
int xllm_index_export(xllm_ingest_t h, int64_t capacity, uint8_t* keys, uint64_t* hbm, uint64_t* dram, uint64_t* ssd,
                      int64_t* n_keys) {
  XLLM_TRY_RC(need_index(h));
  if (!n_keys || capacity < 0 || (capacity > 0 && (!keys || !hbm || !dram || !ssd))) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  std::lock_guard<std::mutex> lock2(*h->index_mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  return h->index->export_all(h->stream, capacity, keys, hbm, dram, ssd, n_keys);
}
int xllm_index_erase(xllm_ingest_t h, const uint8_t* key16) {
  XLLM_TRY_RC(need_index(h));
  if (!key16) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(*h->index_mu);
  if (!owns_key(h, key16)) return XLLM_OK;
  h->index->erase(key16);
  return XLLM_OK;
}
int xllm_index_publish(xllm_ingest_t h) {
  XLLM_TRY_RC(need_index(h));
  std::lock_guard<std::mutex> lock(h->mu);
  std::lock_guard<std::mutex> lock2(*h->index_mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  return h->index->publish(h->stream);
}
int xllm_index_clear_instance(xllm_ingest_t h, int32_t instance_id) {
  XLLM_TRY_RC(need_index(h));
  if (instance_id < 0 || instance_id >= kMaxInstances) {
    set_last_error("xllm_index_clear_instance: invalid instance id %d", instance_id);
    return XLLM_ERR_INVALID_ARG;
  }
  std::lock_guard<std::mutex> lock(h->mu);
  std::lock_guard<std::mutex> lock2(*h->index_mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  return h->index->clear_instance(h->stream, instance_id);
}
int xllm_index_stats(xllm_ingest_t h, int64_t* live_keys, int64_t* tombstones, int64_t* rebuilds) {
  XLLM_TRY_RC(need_index(h));
  std::lock_guard<std::mutex> lock2(*h->index_mu);
  if (live_keys) *live_keys = h->index->live_keys();
  if (tombstones) *tombstones = h->index->tombstones();
  if (rebuilds) *rebuilds = h->index->rebuilds();
  return XLLM_OK;
}
int xllm_index_size(xllm_ingest_t h, int64_t* n_keys) {
  XLLM_TRY_RC(need_index(h));
  if (!n_keys) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  return h->index->size(h->stream, n_keys);
}
int xllm_index_get(xllm_ingest_t h, const uint8_t* key16, uint64_t masks3[3], int32_t* found) {
  XLLM_TRY_RC(need_index(h));
  if (!key16 || !masks3 || !found) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  std::lock_guard<std::mutex> lock2(*h->index_mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  int f = 0;
  int rc = h->index->get(h->stream, key16, masks3, &f);
  *found = f;
  return rc;
}

int xllm_set_instance(xllm_ingest_t h, int32_t id, int32_t type, int32_t schedulable) {
  if (!h || id < 0 || id >= kMaxInstances || type < 0 || type > 3) {
    set_last_error("xllm_set_instance: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  std::lock_guard<std::mutex> lock(*h->index_mu);
  InstanceTable& t = *h->inst_host;
  const uint64_t bit = 1ull << id;
  t.schedulable = schedulable ? (t.schedulable | bit) : (t.schedulable & ~bit);
  t.decode_type = type == 2 ? (t.decode_type | bit) : (t.decode_type & ~bit);
  h->inst_dirty = true;
  return XLLM_OK;
}
int xllm_set_load_metrics(xllm_ingest_t h, int32_t id, int32_t has_metrics, uint64_t waiting, float usage) {
  if (!h || id < 0 || id >= kMaxInstances) {
    set_last_error("xllm_set_load_metrics: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  std::lock_guard<std::mutex> lock(*h->index_mu);
  InstanceTable& t = *h->inst_host;
  const uint64_t bit = 1ull << id;
  t.has_metrics = has_metrics ? (t.has_metrics | bit) : (t.has_metrics & ~bit);
  t.waiting[id] = waiting;
  t.usage[id] = usage;
  h->inst_dirty = true;
  return XLLM_OK;
}

// uploads the instance view if it changed (always: clones share the host copy, so it is cheap to resend)
static int sync_instances(xllm_ingest_t h, cudaStream_t s) {
  std::lock_guard<std::mutex> lock(*h->index_mu);
  XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_inst, h->inst_host.get(), sizeof(InstanceTable), cudaMemcpyHostToDevice, s));
  h->inst_dirty = false;
  return XLLM_OK;
}

int xllm_index_probe_device(xllm_ingest_t h, const uint8_t* d_keys, int64_t n_keys, uint64_t* d_masks3,
                            void* cuda_stream) {
  XLLM_TRY_RC(need_index(h));
  if (n_keys < 0 || (n_keys > 0 && (!d_keys || !d_masks3))) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : h->stream;
  h->index->begin_read();
  const cudaError_t e = h->index->probe(d_keys, n_keys, d_masks3, s);
  h->index->end_read(h->index_read_ev, s);
  XLLM_CUDA_TRY(e);
  return XLLM_OK;
}

int xllm_score_route_device(xllm_ingest_t h, int32_t n_req, const uint64_t* d_masks3, const int64_t* d_key_start,
                            const int32_t* d_n_blocks, xllm_match_out* d_match, xllm_routing_out* d_routing,
                            void* cuda_stream) {
  if (!h || n_req < 0 || (n_req > 0 && (!d_masks3 || !d_key_start || !d_n_blocks))) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : h->stream;
  XLLM_TRY_RC(sync_instances(h, s));
  XLLM_CUDA_TRY(score_route_launch(d_masks3, d_key_start, d_n_blocks, n_req, h->d_inst,
                                   reinterpret_cast<MatchOut*>(d_match), reinterpret_cast<RoutingOut*>(d_routing), s));
  return XLLM_OK;
}

int xllm_match_route_device(xllm_ingest_t h, int32_t n_req, const uint8_t* d_keys, int64_t n_keys_total,
                            const int64_t* d_key_start, const int32_t* d_n_blocks, xllm_match_out* d_match,
                            xllm_routing_out* d_routing, void* cuda_stream) {
  XLLM_TRY_RC(need_index(h));
  if (n_req < 0 || n_keys_total < 0 || (n_req > 0 && (!d_key_start || !d_n_blocks)) || (n_keys_total > 0 && !d_keys))
    return XLLM_ERR_INVALID_ARG;
  if (n_req == 0 && !h->shard) return XLLM_OK;   // a sharded round is collective: an empty rank still takes part
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : h->stream;
  XLLM_TRY_RC(sync_instances(h, s));   // takes index_mu: before begin_read, never inside (publish: index_mu -> writer lock)
  if (h->shard)   // collective; synchronises `s`
    return h->shard->match_route(*h->index, h->index_read_ev, d_keys, d_key_start, d_n_blocks, n_req, n_keys_total,
                                 h->d_inst, reinterpret_cast<MatchOut*>(d_match),
                                 reinterpret_cast<RoutingOut*>(d_routing), s);
  h->index->begin_read();
  const cudaError_t e = h->index->match_route(d_keys, d_key_start, d_n_blocks, n_req, h->d_inst,
                                              reinterpret_cast<MatchOut*>(d_match),
                                              reinterpret_cast<RoutingOut*>(d_routing), s);
  h->index->end_read(h->index_read_ev, s);
  XLLM_CUDA_TRY(e);
  return XLLM_OK;
}

int xllm_match_route(xllm_ingest_t h, int32_t n_req, const uint8_t* keys, int64_t n_keys_total,
                     const int64_t* key_start, const int32_t* n_blocks, xllm_match_out* match,
                     xllm_routing_out* routing) {
  XLLM_TRY_RC(need_index(h));
  if (n_req < 0 || n_keys_total < 0 || (n_req > 0 && (!key_start || !n_blocks)) || (n_keys_total > 0 && !keys))
    return XLLM_ERR_INVALID_ARG;
  if (n_req == 0 && !h->shard) return XLLM_OK;   // a sharded round is collective: an empty rank still takes part
  for (int32_t r = 0; r < n_req; ++r)
    if (n_blocks[r] < 0 || n_blocks[r] > 65535 || key_start[r] < 0 || key_start[r] + n_blocks[r] > n_keys_total) {
      set_last_error("xllm_match_route: request %d out of bounds", r);
      return XLLM_ERR_INVALID_ARG;
    }
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  XLLM_TRY_RC(h->d_keys.reserve((size_t)n_keys_total * 16 + 64));
  XLLM_TRY_RC(h->d_key_start.reserve((size_t)n_req * 8 + 8));
  XLLM_TRY_RC(h->d_nblk.reserve((size_t)n_req * 4 + 8));
  XLLM_TRY_RC(h->d_match.reserve((size_t)n_req * sizeof(MatchOut) + 8));
  XLLM_TRY_RC(h->d_routing.reserve((size_t)n_req * sizeof(RoutingOut) + 8));
  if (n_keys_total)
    XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_keys.p, keys, (size_t)n_keys_total * 16, cudaMemcpyHostToDevice, s));
  if (n_req) {
    XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_key_start.p, key_start, (size_t)n_req * 8, cudaMemcpyHostToDevice, s));
    XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_nblk.p, n_blocks, (size_t)n_req * 4, cudaMemcpyHostToDevice, s));
  }
  XLLM_TRY_RC(sync_instances(h, s));
  if (h->shard) {
    XLLM_TRY_RC(h->shard->match_route(*h->index, h->index_read_ev, h->d_keys.as<uint8_t>(), h->d_key_start.as<int64_t>(),
                                   h->d_nblk.as<int32_t>(), n_req, n_keys_total, h->d_inst, h->d_match.as<MatchOut>(),
                                   h->d_routing.as<RoutingOut>(), s));
  } else {
    h->index->begin_read();
    const cudaError_t me = h->index->match_route(h->d_keys.as<uint8_t>(), h->d_key_start.as<int64_t>(),
                                                 h->d_nblk.as<int32_t>(), n_req, h->d_inst,
                                                 h->d_match.as<MatchOut>(), h->d_routing.as<RoutingOut>(), s);
    h->index->end_read(h->index_read_ev, s);
    XLLM_CUDA_TRY(me);
  }
  if (match && n_req)
    XLLM_CUDA_TRY(cudaMemcpyAsync(match, h->d_match.p, (size_t)n_req * sizeof(MatchOut), cudaMemcpyDeviceToHost, s));
  if (routing && n_req)
    XLLM_CUDA_TRY(
        cudaMemcpyAsync(routing, h->d_routing.p, (size_t)n_req * sizeof(RoutingOut), cudaMemcpyDeviceToHost, s));
  XLLM_CUDA_TRY(cudaStreamSynchronize(s));
  return XLLM_OK;
}

int xllm_tokenizer_probe(const char* tokenizer_path, xllm_tokenizer_info* out) {
  if (!tokenizer_path || !out) {
    set_last_error("xllm_tokenizer_probe: null argument");
    return XLLM_ERR_INVALID_ARG;
  }
  SpTables t;
  const int rc = load_tokenizer_tables(tokenizer_path, &t);
  if (rc != XLLM_OK) {
    set_last_error("tokenizer %s: %s", tokenizer_path, t.error.c_str());
    return rc;
  }
  out->n_pieces = (int32_t)t.n_pieces;
  out->n_symbols = (int32_t)t.n_syms;
  out->n_pair_slots = (int32_t)t.pair_table.size();
  int32_t used = 0;
  for (const auto& e : t.pair_table) used += e.a != kEmptyKey;
  out->n_pairs = used;
  out->split_mode = t.split_mode;
  out->max_unit_out = (int32_t)t.max_unit_out;
  out->byte_fallback = t.byte_fallback;
  out->unk_id = t.unk_id;
  out->trie_units = (int32_t)t.trie.size();
  {
    // probe statistics of the pair table under the device's slot function

    const uint32_t n = (uint32_t)t.pair_table.size();
    uint64_t total = 0;
    uint32_t mx = 0, cnt = 0;
    for (uint32_t i = 0; i < n; ++i) {
      const auto& e = t.pair_table[i];
      if (e.a == kEmptyKey) continue;
      const uint32_t home = sp_pair_slot_fwd(e.a, e.b, n);
      const uint32_t d = ((i + n - home) & (n - 1)) + 1;
      total += d;
      mx = d > mx ? d : mx;
      ++cnt;
    }
    out->avg_probe_x100 = cnt ? (int32_t)(total * 100 / cnt) : 0;
    out->max_probe = (int32_t)mx;
  }
  return XLLM_OK;
}

int xllm_vocab_size(xllm_ingest_t h, int32_t* out) {
  if (!h || !out) return XLLM_ERR_INVALID_ARG;
  if (!h->sp_tables) {
    set_last_error("handle has no tokenizer");
    return XLLM_ERR_UNSUPPORTED;
  }
  *out = h->sp_tables->vocab_size_override >= 0 ? h->sp_tables->vocab_size_override : (int32_t)h->sp_tables->n_pieces;
  return XLLM_OK;
}

int xllm_encode_batch_device(xllm_ingest_t h, int32_t n_req, const uint8_t* d_text, const int64_t* d_offsets,
                             int32_t* d_ids, int64_t ids_stride, int32_t* d_n_ids, int32_t* d_status,
                             void* cuda_stream) {
  if (!h || n_req < 0 || ids_stride < 0 || (n_req > 0 && (!d_offsets || !d_ids || !d_n_ids || !d_status))) {
    set_last_error("xllm_encode_batch_device: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  if (!h->sp_dev) {
    set_last_error("handle has no tokenizer (tokenizer_path was not set)");
    return XLLM_ERR_UNSUPPORTED;
  }
  if (n_req == 0) return XLLM_OK;
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : h->stream;
  SpMemo memo;
  SpEncodePlan plan;
  XLLM_TRY_RC(encode_reserve(h, n_req, &h->d_defer, &h->d_memo, &h->memo_age, &memo, &plan));
  SpLaunchOpts opts;
  opts.nfc_verify = plan.nfc_verify;
  XLLM_CUDA_TRY(sp_encode_launch(h->sp_dev->dev(), d_text, d_offsets, n_req, d_ids, ids_stride, d_n_ids, d_status,
                                 h->d_task_counter + 4, h->d_defer.p, s, memo, opts));
  return XLLM_OK;
}

static int encode_batch_impl(xllm_ingest_t h, int32_t n_req, const uint8_t* text, const int64_t* offsets, int32_t* ids,
                             int64_t ids_stride, int32_t* n_ids, int32_t* status, uint64_t* warp_ns, int32_t warp_cap,
                             int32_t* n_warps) {
  if (!h || n_req < 0 || ids_stride < 0 || (n_req > 0 && (!offsets || !n_ids || !status)) ||
      (n_req > 0 && ids_stride > 0 && !ids && !warp_ns)) {
    set_last_error("xllm_encode_batch: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  if (!h->sp_dev) {
    set_last_error("handle has no tokenizer (tokenizer_path was not set)");
    return XLLM_ERR_UNSUPPORTED;
  }
  if (n_req == 0) return XLLM_OK;
  for (int32_t r = 0; r < n_req; ++r) {
    if (offsets[r + 1] < offsets[r] || offsets[r] < 0 || offsets[r + 1] - offsets[r] > 0x7fffffffLL) {
      set_last_error("xllm_encode_batch: bad offsets at request %d", r);
      return XLLM_ERR_INVALID_ARG;
    }
  }
  const size_t text_bytes = (size_t)(offsets[n_req] - offsets[0]);
  if (text_bytes > 0 && !text) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  XLLM_TRY_RC(h->d_text.reserve(text_bytes + 16));
  XLLM_TRY_RC(h->d_offsets.reserve((size_t)(n_req + 1) * 8));
  XLLM_TRY_RC(h->d_ids.reserve((size_t)n_req * (size_t)ids_stride * 4 + 16));
  XLLM_TRY_RC(h->d_n_ids.reserve((size_t)n_req * 4));
  XLLM_TRY_RC(h->d_status.reserve((size_t)n_req * 4));
  cudaStream_t s = h->stream;
  SpMemo memo;
  SpEncodePlan plan;
  XLLM_TRY_RC(encode_reserve(h, n_req, &h->d_defer, &h->d_memo, &h->memo_age, &memo, &plan));
  // offsets are rebased on the device copy of the text: ship them relative to offsets[0]
  if (text_bytes)
    XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_text.p, text + offsets[0], text_bytes, cudaMemcpyHostToDevice, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_offsets.p, offsets, (size_t)(n_req + 1) * 8, cudaMemcpyHostToDevice, s));
  SpLaunchOpts opts;
  opts.nfc_verify = plan.nfc_verify;
  const int grid = plan.warp_ns;
  if (warp_ns) {   // diagnostics: per-warp busy time of the persistent grid
    XLLM_TRY_RC(h->d_masks.reserve((size_t)grid * 8 + 8));
    XLLM_CUDA_TRY(cudaMemsetAsync(h->d_masks.p, 0, (size_t)grid * 8, s));
    opts.warp_ns = h->d_masks.as<unsigned long long>();
  }
  XLLM_CUDA_TRY(sp_encode_launch(h->sp_dev->dev(), h->d_text.as<uint8_t>() - offsets[0], h->d_offsets.as<int64_t>(),
                                 n_req, h->d_ids.as<int32_t>(), ids_stride, h->d_n_ids.as<int32_t>(),
                                 h->d_status.as<int32_t>(), h->d_task_counter + 4, h->d_defer.p, s, memo,
                                 opts));
  if (warp_ns) {
    const int take = grid < warp_cap ? grid : warp_cap;
    if (take > 0) XLLM_CUDA_TRY(cudaMemcpyAsync(warp_ns, h->d_masks.p, (size_t)take * 8, cudaMemcpyDeviceToHost, s));
    if (n_warps) *n_warps = grid;
  }
  if (ids_stride && ids)
    XLLM_CUDA_TRY(cudaMemcpyAsync(ids, h->d_ids.p, (size_t)n_req * (size_t)ids_stride * 4, cudaMemcpyDeviceToHost, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(n_ids, h->d_n_ids.p, (size_t)n_req * 4, cudaMemcpyDeviceToHost, s));
  XLLM_CUDA_TRY(cudaMemcpyAsync(status, h->d_status.p, (size_t)n_req * 4, cudaMemcpyDeviceToHost, s));
  XLLM_CUDA_TRY(cudaStreamSynchronize(s));
  return XLLM_OK;
}

int xllm_encode_batch(xllm_ingest_t h, int32_t n_req, const uint8_t* text, const int64_t* offsets, int32_t* ids,
                      int64_t ids_stride, int32_t* n_ids, int32_t* status) {
  return encode_batch_impl(h, n_req, text, offsets, ids, ids_stride, n_ids, status, nullptr, 0, nullptr);
}
int xllm_encode_batch_profile(xllm_ingest_t h, int32_t n_req, const uint8_t* text, const int64_t* offsets,
                              int64_t ids_stride, int32_t* n_ids, int32_t* status, uint64_t* warp_ns, int32_t warp_cap,
                              int32_t* n_warps) {
  if (!warp_ns || warp_cap <= 0) return XLLM_ERR_INVALID_ARG;
  return encode_batch_impl(h, n_req, text, offsets, nullptr, ids_stride, n_ids, status, warp_ns, warp_cap, n_warps);
}

}  // extern "C"
