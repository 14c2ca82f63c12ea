// reference_adaptors.h — the reference-side bindings a maintainer drops into xllm-service to put the
// H100 path behind its existing seams.  It includes the reference's OWN headers (tokenizer/tokenizer.h,
// common/slice.h, common/types.h, scheduler/loadbalance_policy/loadbalance_policy.h) and is compiled against them,
// unmodified, by oracle/build_ref.sh into oracle/_ref/reference_seams_test (tests/cpp/reference_seams_main.cc,
// run on the GPU by tests/test_gpu_reference_seams.py).  See INTEGRATION.md.
//
//   GpuTokenizer          : a 4th Tokenizer backend (tokenizer/tokenizer.h:28-46), selected in
//                           TokenizerFactory::create_tokenizer (tokenizer_factory.cpp:9-32); requests the device
//                           path refuses (XLLM_ERR_UNSUPPORTED / XLLM_ERR_CAPACITY) go to a wrapped stock Tokenizer
//   GpuGlobalKVCacheIndex : the calls Scheduler / CacheAwareRouting make on GlobalKVCacheMgr
//                           (global_kvcache_mgr.h:39-45) + name <-> instance-id bookkeeping
//   GpuCacheAwareRouting  : LoadBalancePolicy (loadbalance_policy.h:24-35) — select_instances_pair
//                           (cache_aware_routing.cpp:22-57) computed on the device, names written to Request::routing
#pragma once
#include <memory>
#include <mutex>
#include <optional>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "common/slice.h"
#include "common/types.h"
#include "request/request.h"
#include "scheduler/loadbalance_policy/loadbalance_policy.h"
#include "tokenizer/tokenizer.h"
#include "tokenizer/tokenizers/tokenizers.h"   // the reference's own FFI header; libxllm_ingest.so serves its symbols
#include "index_snapshot.h"
#include "xllm_ingest.h"     // this repo: include/xllm_ingest.h
#include "xllm_rpc_service.pb.h"

namespace xllm_service {

// ---------------------------------------------------------------------------- tokenizer
class GpuTokenizer final : public Tokenizer {
 public:
  // `fallback`: the stock backend TokenizerFactory would have built for this directory (may be null).  It serves
  // the requests the device path refuses by contract — a tokenizer.json with `normalizer: NFC` and a text that is
  // not provably NFC already, a single pre-token longer than the device scratch — so that no request the
  // reference would have tokenised fails (Scheduler::schedule fails a request whose encode returns false,
  // scheduler.cpp:129-132).
  GpuTokenizer(const std::string& tokenizer_dir, int device, int32_t block_size, uint32_t seed,
               std::unique_ptr<Tokenizer> fallback = nullptr)
      : dir_(tokenizer_dir), fallback_(std::move(fallback)) {
    xllm_ingest_config cfg{};
    cfg.tokenizer_path = dir_.c_str();
    cfg.block_size = block_size;
    cfg.xxh3_seed = seed;
    cfg.device = device;
    CHECK_EQ(xllm_ingest_create(&cfg, &h_), XLLM_OK) << xllm_last_error();
    // normalizer NFC: serve every request that is in NFC on the device; only text NFC would change goes to fallback_
    xllm_set_nfc_policy(h_, XLLM_NFC_VERIFY);
    legacy_ = tokenizers_new_from_path(dir_.c_str());  // decode / vocabulary queries
  }
  GpuTokenizer(xllm_ingest_t cloned, const std::string& dir, std::unique_ptr<Tokenizer> fallback)
      : h_(cloned), dir_(dir), fallback_(std::move(fallback)) {
    legacy_ = tokenizers_new_from_path(dir_.c_str());
  }
  ~GpuTokenizer() override {
    tokenizers_free(legacy_);
    xllm_ingest_destroy(h_);
  }

  // Appends, like the SentencePiece / tiktoken backends (sentencepiece_tokenizer.cpp:122-126).  Returns false
  // only where the reference itself has no answer (malformed UTF-8 under tokenizer.json: the Rust shim panics,
  // lib.rs:91) or when a refused request has no fallback.
  bool encode(const std::string_view& text, std::vector<int32_t>* ids) const override {
    const int64_t off[2] = {0, (int64_t)text.size()};
    std::vector<int32_t> buf(text.size() + 16);
    int32_t n = 0, st = 0;
    for (int attempt = 0; attempt < 2; ++attempt) {
      if (xllm_encode_batch(h_, 1, reinterpret_cast<const uint8_t*>(text.data()), off, buf.data(),
                            (int64_t)buf.size(), &n, &st) != XLLM_OK)
        return delegate(text, ids);
      if (st != XLLM_ENC_TRUNCATED) break;
      buf.resize((size_t)n);
    }
    if (st == XLLM_ERR_UNSUPPORTED || st == XLLM_ERR_CAPACITY) return delegate(text, ids);
    if (st != XLLM_OK) return false;
    ids->insert(ids->end(), buf.begin(), buf.begin() + n);
    return true;
  }
  std::string decode(const Slice<int32_t>& ids, bool skip_special_tokens) const override {
    const char* data = nullptr;
    size_t len = 0;
    tokenizers_decode(legacy_, reinterpret_cast<const uint32_t*>(ids.data()), ids.size(), skip_special_tokens, &data,
                      &len);
    return {data, len};
  }
  std::optional<int32_t> token_to_id(const std::string_view& token) const override {
    int32_t id = -1;
    tokenizers_token_to_id(legacy_, token.data(), token.size(), &id);
    return id == -1 ? std::nullopt : std::optional<int32_t>(id);
  }
  std::string id_to_token(int32_t id) const override {
    const char* data = nullptr;
    size_t len = 0;
    tokenizers_id_to_token(legacy_, (uint32_t)id, &data, &len);
    return {data, len};
  }
  size_t vocab_size() const override {
    size_t n = 0;
    tokenizers_get_vocab_size(legacy_, &n);
    return n;
  }
  // Cheap: shares the device tables (the reference's clones reload the model from disk,
  // sentencepiece_tokenizer.cpp:254-256); the fallback is cloned its own way.
  std::unique_ptr<Tokenizer> clone() const override {
    xllm_ingest_t c = nullptr;
    CHECK_EQ(xllm_ingest_clone(h_, &c), XLLM_OK) << xllm_last_error();
    return std::make_unique<GpuTokenizer>(c, dir_, fallback_ ? fallback_->clone() : nullptr);
  }
  xllm_ingest_t handle() const { return h_; }
  size_t delegated() const { return delegated_; }   // requests served by the stock tokenizer so far

 private:
  bool delegate(const std::string_view& text, std::vector<int32_t>* ids) const {
    if (!fallback_) return false;
    ++delegated_;
    return fallback_->encode(text, ids);
  }
  xllm_ingest_t h_ = nullptr;
  TokenizerHandle legacy_ = nullptr;
  std::string dir_;
  std::unique_ptr<Tokenizer> fallback_;
  mutable size_t delegated_ = 0;   // a Tokenizer is per-thread (scheduler.cpp:274-277): no atomics needed
};

// ---------------------------------------------------------------------------- prefix index
class GpuGlobalKVCacheIndex {
 public:
  explicit GpuGlobalKVCacheIndex(xllm_ingest_t h) : h_(h), names_(XLLM_MAX_INSTANCES) {}

  // name -> bit position of the tier masks.  -1 when all XLLM_MAX_INSTANCES positions are taken (the caller drops
  // the event / the instance stays unroutable through this policy) — never aborts.  Positions are recycled by
  // release_instance().
  int instance_id(const std::string& name) {
    {
      std::shared_lock<std::shared_mutex> l(mu_);
      auto it = ids_.find(name);
      if (it != ids_.end()) return it->second;
    }
    std::unique_lock<std::shared_mutex> l(mu_);
    auto it = ids_.find(name);
    if (it != ids_.end()) return it->second;
    for (int i = 0; i < XLLM_MAX_INSTANCES; ++i)
      if (!used_[i]) {
        used_[i] = true;
        names_[i] = name;
        ids_[name] = i;
        return i;
      }
    LOG(ERROR) << "GpuGlobalKVCacheIndex: more than " << XLLM_MAX_INSTANCES << " live instances; '" << name
               << "' is not indexed";
    return -1;
  }
  int find_instance(const std::string& name) const {
    std::shared_lock<std::shared_mutex> l(mu_);
    auto it = ids_.find(name);
    return it == ids_.end() ? -1 : it->second;
  }
  std::string name_of(int id) const {
    std::shared_lock<std::shared_mutex> l(mu_);
    return id >= 0 && id < XLLM_MAX_INSTANCES && used_[id] ? names_[id] : std::string();
  }
  // An instance left the cluster (InstanceMgr::deregister_instance): forget its load metrics, clear its bit in
  // every index entry (entries left empty are erased) and make the position reusable.
  bool release_instance(const std::string& name) {
    std::unique_lock<std::shared_mutex> l(mu_);
    auto it = ids_.find(name);
    if (it == ids_.end()) return true;
    const int id = it->second;
    xllm_set_load_metrics(h_, id, 0, 0, 0.f);
    xllm_set_instance(h_, id, 0, 0);
    if (xllm_index_clear_instance(h_, id) != XLLM_OK) return false;
    ids_.erase(it);
    used_[id] = false;
    names_[id].clear();
    return true;
  }

  // InstanceMgr's view consumed by get_load_metrics (instance_mgr.cpp:287-359)
  bool set_instance(const std::string& name, InstanceType type, bool schedulable) {
    const int id = instance_id(name);
    return id >= 0 && xllm_set_instance(h_, id, (int32_t)type, schedulable ? 1 : 0) == XLLM_OK;
  }
  bool set_load_metrics(const std::string& name, const LoadMetrics& m) {
    const int id = instance_id(name);
    return id >= 0 &&
           xllm_set_load_metrics(h_, id, 1, m.waiting_requests_num, m.gpu_cache_usage_perc) == XLLM_OK;
  }
  bool clear_load_metrics(const std::string& name) {
    const int id = find_instance(name);
    return id < 0 || xllm_set_load_metrics(h_, id, 0, 0, 0.f) == XLLM_OK;
  }

  // GlobalKVCacheMgr::record_updated_kvcaches (global_kvcache_mgr.cpp:177-225)
  void record_updated_kvcaches(const std::string& instance_name, const proto::KvCacheEvent& e) {
    const int id = instance_id(instance_name);
    if (id < 0) return;
    std::string s, o, r;
    for (int i = 0; i < e.stored_cache_size(); ++i) s.append(e.stored_cache(i).data(), XLLM_KEY_BYTES);
    for (int i = 0; i < e.offload_cache_size(); ++i) o.append(e.offload_cache(i).data(), XLLM_KEY_BYTES);
    for (int i = 0; i < e.removed_cache_size(); ++i) r.append(e.removed_cache(i).data(), XLLM_KEY_BYTES);
    xllm_index_apply(h_, id, reinterpret_cast<const uint8_t*>(s.data()), s.size() / 16,
                     reinterpret_cast<const uint8_t*>(o.data()), o.size() / 16,
                     reinterpret_cast<const uint8_t*>(r.data()), r.size() / 16);
  }
  // GlobalKVCacheMgr::upload_kvcache's local effect (:227-247); the etcd write stays where it is
  bool upload_kvcache() { return xllm_index_publish(h_) == XLLM_OK; }

  // The table as the pairs the master keeps under XLLM:CACHE: (etcd_client.cpp:122-137), e.g. to seed a new etcd
  // cluster or to hand the index to a freshly elected master; host/index_snapshot.h.
  bool snapshot(const std::string& namespace_prefix, std::vector<xllm_host::CacheKv>* out) {
    std::shared_lock<std::shared_mutex> l(mu_);
    return xllm_host::snapshot_index(h_, namespace_prefix, names_, out) == XLLM_OK;
  }
  // The constructor's start-up load (:47-51) and the replica watch (:133-175): the pairs of one listing / one
  // watch response (empty value = DELETE).  prefix_len = size of namespace + "XLLM:CACHE:".
  bool apply_etcd_pairs(const std::vector<xllm_host::CacheKv>& kvs, size_t prefix_len) {
    size_t skipped = 0;
    const int rc = xllm_host::apply_etcd_pairs(
        h_, prefix_len, kvs, [this](const std::string& n) { return instance_id(n); }, &skipped);
    if (skipped) LOG(ERROR) << skipped << " XLLM:CACHE pairs could not be parsed";
    return rc == XLLM_OK;
  }

  // GlobalKVCacheMgr::match (:73-131) + CacheAwareRouting's decision for one request (the batch path goes through
  // IngestBatcher).  `routing` may be null.
  bool match(const Slice<int32_t>& token_ids, int32_t block_size, OverlapScores* out,
             xllm_routing_out* routing = nullptr) {
    const size_t nb = token_ids.size() / block_size;
    std::vector<uint8_t> keys(16 * (nb ? nb : 1));
    const int64_t zero = 0;
    const int32_t n_tok = (int32_t)token_ids.size(), n_blk = (int32_t)nb;
    if (nb && xllm_hash_blocks(h_, 1, token_ids.data(), n_tok, &zero, &n_tok, keys.data(), (int64_t)nb, &zero) !=
                  XLLM_OK)
      return false;
    xllm_match_out m{};
    if (xllm_match_route(h_, 1, keys.data(), (int64_t)nb, &zero, &n_blk, &m, routing) != XLLM_OK) return false;
    if (out == nullptr || nb == 0) return true;   // n_tokens == 0: OverlapScores untouched (:77-79)
    out->max_block_num = m.max_block_num;
    out->max_matched_block_num = m.max_matched_block_num;
    std::shared_lock<std::shared_mutex> l(mu_);
    for (int i = 0; i < XLLM_MAX_INSTANCES; ++i) {
      if (!((m.instances >> i) & 1) || !used_[i]) continue;
      out->instances.insert(names_[i]);
      if (m.hbm_instance_score[i]) out->hbm_instance_score[names_[i]] = m.hbm_instance_score[i];
      if (m.dram_instance_score[i]) out->dram_instance_score[names_[i]] = m.dram_instance_score[i];
      if (m.ssd_instance_score[i]) out->ssd_instance_score[names_[i]] = m.ssd_instance_score[i];
    }
    return true;
  }

 private:
  xllm_ingest_t h_;
  mutable std::shared_mutex mu_;
  std::unordered_map<std::string, int> ids_;
  std::vector<std::string> names_;          // fixed size: readers index it under the shared lock
  bool used_[XLLM_MAX_INSTANCES] = {};
};

// ---------------------------------------------------------------------------- routing policy
// CacheAwareRouting (cache_aware_routing.h:24-46) with match + get_load_metrics + cost_function evaluated by
// score_route on the device.  The instance view is pushed into the index adaptor by whoever updates InstanceMgr
// (set_instance / set_load_metrics above), so select_instances_pair does not read InstanceMgr at all; the
// base-class pointer is kept only because LoadBalancePolicy's constructor takes one.
class GpuCacheAwareRouting final : public LoadBalancePolicy {
 public:
  GpuCacheAwareRouting(std::shared_ptr<InstanceMgr> instance_mgr, std::shared_ptr<GpuGlobalKVCacheIndex> index,
                       int32_t block_size)
      : LoadBalancePolicy(instance_mgr), index_(std::move(index)), block_size_(block_size) {}

  // cache_aware_routing.cpp:22-57: false iff no prefill-side instance is available; a side whose candidates all
  // score <= MIN_SCORE keeps an empty name, as in the reference (:65,80).
  bool select_instances_pair(std::shared_ptr<Request> request) override {
    xllm_routing_out r{};
    Slice<int32_t> token_ids(request->token_ids.data(), request->token_ids.size());
    if (!index_->match(token_ids, block_size_, nullptr, &r)) return false;
    if (!r.ok) return false;
    if (r.prefill_id >= 0) request->routing.prefill_name = index_->name_of(r.prefill_id);
    if (r.decode_id >= 0) request->routing.decode_name = index_->name_of(r.decode_id);
    return true;
  }

 private:
  std::shared_ptr<GpuGlobalKVCacheIndex> index_;
  int32_t block_size_;
};

}  // namespace xllm_service
