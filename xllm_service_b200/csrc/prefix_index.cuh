// prefix_index.cuh — device-resident global prefix-cache index + match + cache-aware routing.
//
// Device replacement for
//   XXH3KeyCacheMap / CacheLocations      xllm_service/common/types.h:38-41,320-365
//   GlobalKVCacheMgr::match + set_score   xllm_service/scheduler/managers/global_kvcache_mgr.cpp:59-131
//   record_updated_kvcaches               global_kvcache_mgr.cpp:177-225
//   upload_kvcache (local effect)         global_kvcache_mgr.cpp:227-247
//   update_kvcache (replica PUT/DELETE)   global_kvcache_mgr.cpp:133-175
//   InstanceMgr::get_load_metrics         xllm_service/scheduler/managers/instance_mgr.cpp:287-359
//   CacheAwareRouting::cost_function      xllm_service/scheduler/loadbalance_policy/cache_aware_routing.cpp:59-85
//
// Layout in HBM: open-addressing table of 64-byte slots
//   { key low64, key high64, state, hbm mask | dram mask, ssd mask }   (instance sets -> 64-bit masks; two sectors)
// sized to >= 2x the configured key capacity (power of two), linear probing from the key's low64.
//
// Readers and writers (the reference: shared_lock in match, unique_lock in upload_kvcache / update_kvcache,
// global_kvcache_mgr.cpp:83,165,234): handles that share one PrefixIndex read it from their own streams.  A reader
// brackets the ENQUEUE of its kernels with begin_read() / end_read(event, stream); publish / clear_instance / rebuild
// take the lock exclusively, make their stream wait for every registered reader event, mutate, and synchronise
// before releasing — so a probe sees the table either before or after a publish, never in between.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <shared_mutex>
#include <unordered_map>
#include <vector>

namespace xllm {

constexpr int kMaxInstances = 64;

// Field order = sector order: key, state and the HBM mask share the first 32-byte sector (what a probe that does not
// match reads); DRAM still serves the whole 64-byte line (DESIGN.md §6).
struct IndexSlot {
  uint64_t klo, khi;
  uint32_t state;  // 0 empty, 1 full, 2 tombstone, 3 busy (claimed by an insert, key not yet visible)
  uint32_t pad0;
  uint64_t hbm;
  uint64_t dram, ssd;
  uint64_t pad1[2];
};
static_assert(sizeof(IndexSlot) == 64, "one slot = one 64-byte line");

// What GlobalKVCacheMgr::match fills into OverlapScores (types.h:376-403), per request.
struct MatchOut {
  uint32_t max_block_num;          // floor(n_tokens / block_size)
  uint32_t max_matched_block_num;  // blocks matched before the first miss
  uint64_t instances;              // OverlapScores::instances as a bitmask
  uint16_t hbm_score[kMaxInstances];   // 0 = not in hbm_instance_score
  uint16_t dram_score[kMaxInstances];
  uint16_t ssd_score[kMaxInstances];
};
static_assert(sizeof(MatchOut) == 16 + 3 * 2 * kMaxInstances, "MatchOut layout is part of the C-ABI");

// Routing (types.h:43-55) as instance ids; ok == 0 <=> select_instances_pair returned false.
struct RoutingOut {
  int32_t prefill_id;  // -1: name left empty
  int32_t decode_id;
  int32_t ok;
  float prefill_score;  // best cost_function score (MIN_SCORE = -2 when nothing beat it)
  float decode_score;
};

// Per-instance state the routing epilogue reads (InstanceMgr's instances_ / load_metrics_ views).
struct InstanceTable {
  uint64_t waiting[kMaxInstances];  // LoadMetrics::waiting_requests_num
  float usage[kMaxInstances];       // LoadMetrics::gpu_cache_usage_perc
  uint64_t has_metrics;             // bit i: instance i has an entry in load_metrics_
  uint64_t schedulable;             // bit i: registered and is_instance_schedulable
  uint64_t decode_type;             // bit i: InstanceType::DECODE
};

struct Key128 {
  uint64_t lo, hi;
  bool operator==(const Key128& o) const { return lo == o.lo && hi == o.hi; }
};
struct Key128Hash {
  size_t operator()(const Key128& k) const { return (size_t)(k.lo ^ (k.hi * 0x9E3779B97F4A7C15ull)); }
};

class PrefixIndex {
 public:
  ~PrefixIndex();
  int init(int64_t capacity_keys);
  bool ready() const { return slots_ != nullptr; }

  // ---- staged writes (host), in arrival order per key
  void record(int instance, const uint8_t* stored, size_t ns, const uint8_t* offload, size_t no,
              const uint8_t* removed, size_t nr);
  void put(const uint8_t* key16, uint64_t hbm, uint64_t dram, uint64_t ssd);
  void erase(const uint8_t* key16);
  size_t staged_keys() const { return staged_.size(); }
  // applies every staged op on `stream` and clears the staging area (also when it fails); rebuilds the table in
  // place when tombstones + live keys exceed 70 % of the slots
  int publish(cudaStream_t stream);
  // clears instance `id`'s bit in every entry (entries left empty are erased): the instance left the cluster
  int clear_instance(cudaStream_t stream, int id);
  // live keys / tombstones as of the last publish (host copies, no device round trip)
  int64_t live_keys() const { return live_; }
  int64_t tombstones() const { return tombs_; }
  int64_t rebuilds() const { return rebuilds_; }

  int size(cudaStream_t stream, int64_t* n);
  int get(cudaStream_t stream, const uint8_t* key16, uint64_t masks3[3], int* found);
  // snapshot of every live key with its three masks (order unspecified); *n_out = live keys, also when > cap
  int export_all(cudaStream_t stream, int64_t cap, uint8_t* keys16, uint64_t* hbm, uint64_t* dram, uint64_t* ssd,
                 int64_t* n_out);

  // ---- reads (device pointers, asynchronous on `stream`); call between begin_read() and end_read()
  // masks3[k] = {hbm, dram, ssd} of keys[k], all zero when absent
  cudaError_t probe(const uint8_t* d_keys, int64_t n_keys, uint64_t* d_masks3, cudaStream_t stream) const;
  // GlobalKVCacheMgr::match + CacheAwareRouting in ONE kernel: one warp per request, lane = block, keys probed in
  // waves of 32 blocks, stop after the wave holding the first miss, tier masks kept in registers.
  cudaError_t match_route(const uint8_t* d_keys, const int64_t* d_key_start, const int32_t* d_n_blocks, int n_req,
                          const struct InstanceTable* d_instances, struct MatchOut* d_match,
                          struct RoutingOut* d_routing, cudaStream_t stream) const;

  // owner side of the hash-range-sharded index (shard_exchange.cuh): probe the tuples of `world` received messages
  cudaError_t probe_messages(const uint8_t* d_recv, size_t msg_bytes, int world, uint32_t cap, uint64_t* d_back,
                             cudaStream_t stream) const;

  // ---- reader / writer protocol
  cudaEvent_t register_reader();              // one event per reading handle; null on failure
  void unregister_reader(cudaEvent_t ev);
  void begin_read() { rw_.lock_shared(); }
  void end_read(cudaEvent_t ev, cudaStream_t stream) {
    if (ev) cudaEventRecord(ev, stream);
    rw_.unlock_shared();
  }

  const IndexSlot* slots() const { return slots_; }
  uint64_t mask() const { return n_slots_ - 1; }

 private:
  struct Op {
    uint8_t type;      // 0 stored, 1 offload, 2 removed, 3 assign, 4 erase
    uint8_t instance;
    uint32_t payload;  // assign: index into payload_ (3 masks)
  };
  int wait_for_readers(cudaStream_t stream);   // caller holds rw_ exclusively
  int rebuild(cudaStream_t stream);            // same
  int read_counters(cudaStream_t stream);      // d_counters_ -> live_, tombs_, error flag (returned)
  mutable std::shared_mutex rw_;
  std::mutex ev_mu_;
  std::vector<cudaEvent_t> reader_events_;
  int64_t live_ = 0, tombs_ = 0, rebuilds_ = 0;
  IndexSlot* slots_ = nullptr;
  uint64_t n_slots_ = 0;
  int64_t capacity_ = 0;
  int64_t* d_counters_ = nullptr;  // [0] live keys, [1] insert-list length, [2] error flag, [3] tombstones
  std::unordered_map<Key128, std::vector<Op>, Key128Hash> staged_;
  std::vector<Key128> staged_order_;
  std::vector<uint64_t> payload_;
  void* d_stage_ = nullptr;
  size_t d_stage_cap_ = 0;
};

// One warp per request: first-miss scan over the request's probed masks, per-instance scores,
// then the cache-aware-routing decision.  d_match / d_routing may be null.
cudaError_t score_route_launch(const uint64_t* d_masks3, const int64_t* d_key_start, const int32_t* d_n_blocks,
                               int n_req, const InstanceTable* d_instances, MatchOut* d_match,
                               RoutingOut* d_routing, cudaStream_t stream, const uint32_t* d_pos = nullptr);

}  // namespace xllm
