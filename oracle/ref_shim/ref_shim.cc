// TEST INFRASTRUCTURE — the C entry points of oracle/_ref/libxllm_ref.so.
//
// libxllm_ref.so is the REFERENCE ITSELF for rows a5-a8 / f1 / f3 of the hot path: oracle/build_ref.sh compiles
// these reference files UNMODIFIED, where they lie under the reference checkout's xllm_service/, against the stand-in headers
// in oracle/ref_shim/stubs (glog, gflags, absl::Mutex, an in-memory etcd, hand-written protobuf accessors):
//   common/hash_util.cpp            xxh3_128bits_hash                                   (a5)
//   common/types.h                  CacheLocations JSON, OverlapScores, LoadBalanceInfos (a6, f3)
//   scheduler/managers/global_kvcache_mgr.cpp   match / record_updated_kvcaches / upload_kvcache / update_kvcache (a7, f1)
//   scheduler/etcd_client/etcd_client.cpp       the "XLLM:CACHE:"+key -> JSON wire form  (f3)
//   scheduler/loadbalance_policy/cache_aware_routing.cpp  select_instances_pair + cost_function (a8)
//   common/threadpool.cpp, common/utils.cpp, common/global_gflags.cpp
// and InstanceMgr::get_load_metrics (instance_mgr.cpp:287-359, with is_instance_schedulable :63-66), cut out of
// the reference by line range at build time into oracle/_ref/ (instance_mgr.cpp as a whole needs brpc).
// This file only adapts C arguments to those classes; it restates nothing.  Built with -fno-access-control so the
// adaptors can read GlobalKVCacheMgr::kvcache_infos_ and drain its thread pool.
#include <atomic>
#include <cstring>
#include <future>
#include <memory>
#include <string>

#include "common/global_gflags.h"
#include "common/hash_util.h"
#include "common/options.h"
#include "common/types.h"
#include "scheduler/etcd_client/etcd_client.h"
#include "scheduler/loadbalance_policy/cache_aware_routing.h"
#include "scheduler/managers/global_kvcache_mgr.h"
#include "scheduler/managers/instance_mgr.h"

using namespace xllm_service;

namespace {
struct Ref {
  std::string addr;
  std::shared_ptr<EtcdClient> etcd;
  std::shared_ptr<GlobalKVCacheMgr> mgr;
  std::shared_ptr<InstanceMgr> inst;
  std::shared_ptr<CacheAwareRouting> car;
  bool master;
};
std::atomic<int> g_next{0};

int id_of(const char* const* names, int n, const std::string& s) {
  for (int i = 0; i < n; ++i)
    if (s == names[i]) return i;
  return -1;
}
void drain(Ref* r) {   // wait for update_kvcache's pool task (global_kvcache_mgr.cpp:138)
  std::promise<void> p;
  auto f = p.get_future();
  r->mgr->threadpool_.schedule([&p] { p.set_value(); });
  f.wait();
}
}  // namespace

extern "C" {

// hash_util.cpp:18-45 with FLAGS_xxh3_128bits_seed = seed.  Returns 0.
int ref_xxh3_128bits_hash(const uint8_t* prev16, const int32_t* tokens, size_t n_tokens, uint32_t seed,
                          uint8_t* out16) {
  FLAGS_xxh3_128bits_seed = seed;
  xxh3_128bits_hash(prev16, Slice<int32_t>(tokens, n_tokens), out16);
  return 0;
}

// A GlobalKVCacheMgr (+ InstanceMgr registry + CacheAwareRouting) on its own in-memory etcd ("share" = another
// handle whose etcd to join: a replica of that master when is_master = 0).
void* ref_index_new(uint32_t block_size, uint32_t seed, int is_master, void* share, const char* etcd_namespace) {
  FLAGS_xxh3_128bits_seed = seed;
  Ref* r = new Ref();
  r->addr = share ? ((Ref*)share)->addr : "fake://" + std::to_string(g_next++);
  r->master = is_master != 0;
  r->etcd = std::make_shared<EtcdClient>(r->addr, etcd_namespace ? etcd_namespace : "");
  Options opt;
  opt.block_size((int32_t)block_size);
  opt.xxh3_128bits_seed(seed);
  r->mgr = std::make_shared<GlobalKVCacheMgr>(opt, r->etcd, r->master);
  r->inst = std::make_shared<InstanceMgr>();
  r->car = std::make_shared<CacheAwareRouting>(r->inst, r->mgr);
  return r;
}
void ref_index_free(void* h) {
  Ref* r = (Ref*)h;
  r->car.reset();
  r->mgr.reset();
  r->etcd.reset();
  delete r;
}
long ref_index_size(void* h) {
  Ref* r = (Ref*)h;
  drain(r);
  std::shared_lock<std::shared_mutex> g(r->mgr->kvcache_mutex_);
  return (long)r->mgr->kvcache_infos_.size();
}
// record_updated_kvcaches (global_kvcache_mgr.cpp:177-225) with one KvCacheEvent
void ref_index_record(void* h, const char* name, const uint8_t* stored, size_t ns, const uint8_t* offload, size_t no,
                      const uint8_t* removed, size_t nr) {
  proto::KvCacheEvent ev;
  for (size_t i = 0; i < ns; ++i) ev.add_stored_cache(std::string((const char*)stored + 16 * i, 16));
  for (size_t i = 0; i < no; ++i) ev.add_offload_cache(std::string((const char*)offload + 16 * i, 16));
  for (size_t i = 0; i < nr; ++i) ev.add_removed_cache(std::string((const char*)removed + 16 * i, 16));
  ((Ref*)h)->mgr->record_updated_kvcaches(name, ev);
}
// upload_kvcache (global_kvcache_mgr.cpp:227-247): writes etcd (one watch response for the whole flush) + the map
int ref_index_upload(void* h) {
  Ref* r = (Ref*)h;
  auto st = etcd::fake::store_for(r->addr);
  st->begin_batch();
  bool ok = r->mgr->upload_kvcache();
  st->end_batch();
  return ok ? 1 : 0;
}
void ref_set_rm_missing_is_error(int on) { etcd::SyncClient::rm_missing_is_error() = on != 0; }
// An etcd PUT / DELETE of one cache key by somebody else (what a replica's watch sees): the value is
// CacheLocations::serialize_to_json().dump() (types.h:325-331), the key "XLLM:CACHE:"+16 bytes under the namespace.
void ref_etcd_put(void* h, const uint8_t* key16, const char* const* hbm, int nh, const char* const* dram, int nd,
                  const char* const* ssd, int nsd) {
  Ref* r = (Ref*)h;
  CacheLocations c;
  for (int i = 0; i < nh; ++i) c.hbm_instance_set.insert(hbm[i]);
  for (int i = 0; i < nd; ++i) c.dram_instance_set.insert(dram[i]);
  for (int i = 0; i < nsd; ++i) c.ssd_instance_set.insert(ssd[i]);
  XXH3KeyCacheMap one;
  one.insert_or_assign(XXH3Key(key16), c);   // an all-empty value makes EtcdClient::set issue a DELETE
  r->etcd->set("XLLM:CACHE:", one);
  drain(r);
}
void ref_etcd_put_raw(void* h, const char* key, size_t key_len, const char* value, size_t value_len) {
  Ref* r = (Ref*)h;
  etcd::fake::store_for(r->addr)->put(std::string(key, key_len), std::string(value, value_len));
  drain(r);
}
void ref_etcd_delete(void* h, const uint8_t* key16) {
  Ref* r = (Ref*)h;
  r->etcd->rm("XLLM:CACHE:" + std::string((const char*)key16, 16));
  drain(r);
}
void ref_etcd_batch(void* h, int begin) {
  Ref* r = (Ref*)h;
  auto st = etcd::fake::store_for(r->addr);
  if (begin) st->begin_batch();
  else { st->end_batch(); drain(r); }
}
// Dump of the store under a prefix: for pair i, klen[i]/vlen[i] and the bytes appended to kbuf / vbuf.
// Returns the number of pairs, or -(needed pairs) when a capacity is too small.
long ref_etcd_list(void* h, const char* prefix, char* kbuf, size_t kcap, char* vbuf, size_t vcap, int64_t* klen,
                   int64_t* vlen, size_t max_pairs) {
  Ref* r = (Ref*)h;
  auto st = etcd::fake::store_for(r->addr);
  std::lock_guard<std::recursive_mutex> g(st->mu);
  std::string p(prefix);
  size_t n = 0, ko = 0, vo = 0;
  bool fits = true;
  for (auto it = st->kv.lower_bound(p); it != st->kv.end(); ++it) {
    if (it->first.compare(0, p.size(), p) != 0) break;
    if (n < max_pairs && ko + it->first.size() <= kcap && vo + it->second.size() <= vcap) {
      memcpy(kbuf + ko, it->first.data(), it->first.size());
      memcpy(vbuf + vo, it->second.data(), it->second.size());
      klen[n] = (int64_t)it->first.size();
      vlen[n] = (int64_t)it->second.size();
    } else {
      fits = false;
    }
    ko += it->first.size();
    vo += it->second.size();
    ++n;
  }
  return fits ? (long)n : -(long)n;
}
// kvcache_infos_ lookup: three bitmasks over names[]; 1 if present
int ref_index_get(void* h, const uint8_t* key16, const char* const* names, int n_names, uint64_t* masks3) {
  Ref* r = (Ref*)h;
  drain(r);
  std::shared_lock<std::shared_mutex> g(r->mgr->kvcache_mutex_);
  auto& m = r->mgr->kvcache_infos_;
  auto it = m.find(XXH3Key(key16));
  masks3[0] = masks3[1] = masks3[2] = 0;
  if (it == m.end()) return 0;
  const std::unordered_set<std::string>* sets[3] = {&it->second.hbm_instance_set, &it->second.dram_instance_set,
                                                    &it->second.ssd_instance_set};
  for (int t = 0; t < 3; ++t)
    for (const auto& s : *sets[t]) {
      int id = id_of(names, n_names, s);
      if (id >= 0) masks3[t] |= 1ull << id;
    }
  return 1;
}
// GlobalKVCacheMgr::match (global_kvcache_mgr.cpp:73-131).  scores3: [3][n_names] (0 = absent from the map).
void ref_index_match(void* h, const int32_t* tokens, size_t n_tokens, const char* const* names, int n_names,
                     uint32_t* scores3, uint64_t* instances_mask, uint32_t* max_block_num,
                     uint32_t* max_matched_block_num) {
  Ref* r = (Ref*)h;
  OverlapScores os;
  r->mgr->match(Slice<int32_t>(tokens, n_tokens), &os);
  memset(scores3, 0, sizeof(uint32_t) * 3 * n_names);
  *instances_mask = 0;
  const std::unordered_map<std::string, uint32_t>* maps[3] = {&os.hbm_instance_score, &os.dram_instance_score,
                                                              &os.ssd_instance_score};
  for (int t = 0; t < 3; ++t)
    for (const auto& kv : *maps[t]) {
      int id = id_of(names, n_names, kv.first);
      if (id >= 0) scores3[t * n_names + id] = kv.second;
    }
  for (const auto& s : os.instances) {
    int id = id_of(names, n_names, s);
    if (id >= 0) *instances_mask |= 1ull << id;
  }
  *max_block_num = os.max_block_num;
  *max_matched_block_num = os.max_matched_block_num;
}
// registry = the four InstanceMgr members get_load_metrics reads
void ref_registry_set_instance(void* h, const char* name, int type, int schedulable) {
  InstanceMetaInfo info(name, "rpc://" + std::string(name), (InstanceType)type);
  info.runtime_state = schedulable ? InstanceRuntimeState::ACTIVE : InstanceRuntimeState::SUSPECT;
  ((Ref*)h)->inst->instances_[name] = info;
}
void ref_registry_set_load(void* h, const char* name, uint64_t waiting, float usage) {
  ((Ref*)h)->inst->load_metrics_[name] = LoadMetrics(waiting, usage);
}
void ref_registry_clear_load(void* h, const char* name) { ((Ref*)h)->inst->load_metrics_.erase(name); }
// CacheAwareRouting::select_instances_pair (cache_aware_routing.cpp:22-57): 1/0 = its return value; ids into
// names[] of Request::routing.prefill_name / decode_name (-1 = left empty).
int ref_route_car(void* h, const int32_t* tokens, size_t n_tokens, const char* const* names, int n_names,
                  int* prefill_id, int* decode_id) {
  Ref* r = (Ref*)h;
  auto req = std::make_shared<Request>();
  req->token_ids.assign(tokens, tokens + n_tokens);
  bool ok = r->car->select_instances_pair(req);
  *prefill_id = id_of(names, n_names, req->routing.prefill_name);
  *decode_id = id_of(names, n_names, req->routing.decode_name);
  return ok ? 1 : 0;
}

}  // extern "C"
