// Internal handle behind the C-ABI (include/xllm_ingest.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <memory>

#include "pipeline_schedule.h"
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "prefix_index.cuh"
#include "shard_exchange.cuh"
#include "sp_encode.cuh"
#include "sp_model.h"
#include "xxh3_chain.cuh"

namespace xllm {

// Growable device / pinned-host scratch buffer.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes);
  void release();
  template <typename T>
  T* as() { return static_cast<T*>(p); }
};
struct PinBuf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes);
  void release();
  template <typename T>
  T* as() { return static_cast<T*>(p); }
};

// One in-flight chunk of xllm_ingest_batch: its own stream + device buffers.
constexpr int kPipeSlots = 32;  // upper bound; xllm_ingest::pipe_slots are used
struct PipeSlot {
  cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};  // uploaded / kernels done / downloaded
  bool busy = false;                                // ev[2] of an earlier chunk of this batch is pending
  unsigned int* counters = nullptr;
  DevBuf d_memo;  // this slot's word memo (sp_encode.cuh): cleared by every encode launch on the slot's stream,
                  // or kept for memo_persist_requests requests (xllm_set_memo_policy)
  int64_t memo_age = -1;  // requests encoded since the table was last cleared; -1 = never cleared (must be)
  DevBuf d_defer, d_text, d_offsets, d_ids, d_n_ids, d_status, d_tok_start, d_n_tok, d_key_start, d_n_blocks, d_keys, d_masks,
      d_match, d_routing;
  // segmented requests (xllm_ingest_batch_segments): text pieces encode into ragged temporary rows, then the
  // assemble kernel splices pieces and id spans into the request's row
  DevBuf d_ids16;   // narrow download (xllm_ingest_io::ids_u16)
  DevBuf d_piece_ids, d_piece_n, d_piece_status, d_piece_out_start, d_piece_out_cap, d_seg_len, d_seg_src, d_req_seg,
      d_span;
  int ensure(size_t text_bytes, int n, int64_t ids_stride, int64_t keys_stride, int n_req = -1);
  // host staging of a segmented chunk's small tables: must outlive the asynchronous uploads, so they live in the slot
  std::vector<int64_t> h_piece_out_start, h_seg_src;
  std::vector<int32_t> h_piece_out_cap, h_req_seg;
  void release();
};

}  // namespace xllm

struct xllm_ingest {
  int device = 0;
  int block_size = 128;
  uint32_t seed = 1024;
  int max_batch = 65536;
  int max_tokens = 8192;
  cudaStream_t stream = nullptr;
  std::mutex mu;  // serialises calls on this handle
  xllm::Xxh3Consts xxh;
  unsigned int* d_task_counter = nullptr;
  // tokenizer (shared between clones)
  std::shared_ptr<xllm::SpTables> sp_tables;
  std::shared_ptr<xllm::SpDeviceModel> sp_dev;
  std::string tokenizer_path;
  // prefix index + instance view (shared between clones)
  std::shared_ptr<xllm::PrefixIndex> index;
  std::shared_ptr<std::mutex> index_mu;
  std::shared_ptr<xllm::ShardExchange> shard;      // set when the index is hash-range-sharded (shared by clones)
  cudaEvent_t index_read_ev = nullptr;             // this handle's entry in the index's reader list (prefix_index.cuh)
  std::shared_ptr<xllm::InstanceTable> inst_host;  // host copy
  xllm::InstanceTable* d_inst = nullptr;           // this handle's device copy
  bool inst_dirty = true;
  xllm::DevBuf d_masks, d_match, d_routing, d_nblk;
  // xllm_ingest_batch pipeline
  xllm::PipeSlot pipe[xllm::kPipeSlots];
  cudaStream_t pipe_stream[3] = {nullptr, nullptr, nullptr};  // upload / kernel / download engines of xllm_ingest_batch
  int pipe_slots = 4;
  int last_chunks = 0, last_launches = 0;  // of the most recent xllm_ingest_batch  // chunks in flight (XLLM_PIPE_SLOTS): enough to cover one request-per-warp encode latency
  int pipe_chunk_req = 4096;
  int64_t pipe_chunk_bytes = 96ll << 20;
  // scratch for the host-pointer entry points
  xllm::DevBuf d_text, d_offsets, d_ids, d_n_ids, d_status, d_defer;
  xllm::DevBuf d_memo;      // word memo of the single-launch encode entry points
  int64_t memo_age = -1;    // requests encoded since d_memo was last cleared; -1 = never
  int64_t memo_persist_requests = 0;  // 0: every launch clears its memo; N > 0: a memo is kept until it has seen N requests
  xllm::DevBuf d_arena;     // warm-up scratch of the encode kernel (per handle: launches on one handle are serialised)
  uint32_t memo_slots = 0;  // 0 = memo off
  bool sp_warm = false;     // XLLM_SP_WARM=1: launch the warm-up tokenizer kernels (natural text; sp_encode.cu drain_pass, WARM)
  xllm::DevBuf d_tokens, d_tok_start, d_n_tok, d_keys, d_key_start;
  // sharded xllm_ingest_batch: the whole batch's keys / row descriptors / results stay resident for the one exchange
  xllm::DevBuf d_all_keys, d_all_key_start, d_all_n_blocks, d_all_match, d_all_routing;
};

namespace xllm {
// Plans one sp_encode_launch over n_req rows on handle h and reserves what it needs: the launch scratch, the word memo
// table and the warm-up arena.  memo_buf / memo_age: the handle's or the pipeline slot's table and its age
// (xllm_set_memo_policy), which this launch advances.  Fills *memo for the launch.
int encode_reserve(xllm_ingest* h, int n_req, DevBuf* scratch, DevBuf* memo_buf, int64_t* memo_age, SpMemo* memo,
                   SpEncodePlan* plan);
}  // namespace xllm
