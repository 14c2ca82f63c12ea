// The drop-in boundary, proven by compiling the reference's own files against it (built by oracle/build_ref.sh into
// oracle/_ref/reference_seams_test, because it needs the reference checkout's headers; run on the GPU by
// tests/test_gpu_reference_seams.py):
//   fast  : the reference's tokenizer/fast_tokenizer.cpp, UNMODIFIED, linked against libxllm_ingest.so — its
//           FastTokenizer class (fast_tokenizer.h) drives tokenizers_new_from_path / _encode / _decode /
//           _token_to_id / _id_to_token / _get_vocab_size / _free exactly as in the service;
//   gpu   : host/reference_adaptors.h's GpuTokenizer, a subclass of the reference's real Tokenizer
//           (tokenizer/tokenizer.h:28-46), with a stock tokenizer behind it for refused requests;
//   route : GpuGlobalKVCacheIndex + GpuCacheAwareRouting (a real LoadBalancePolicy subclass,
//           loadbalance_policy.h:24-35) against the reference's own GlobalKVCacheMgr + CacheAwareRouting
//           (oracle/_ref/libxllm_ref.so) fed the same KvCacheEvents, instance view and requests.
// Output: one line per case for the Python side to compare with goldens / the oracle; "OK" last.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <random>
#include <string>
#include <vector>

#include "common/global_gflags.h"
#include "scheduler/loadbalance_policy/cache_aware_routing.h"
#include "scheduler/managers/global_kvcache_mgr.h"
#include "tokenizer/fast_tokenizer.h"
#include "reference_adaptors.h"

using namespace xllm_service;

static std::vector<std::string> read_cases(const char* path) {   // u32 length + bytes, repeated
  std::vector<std::string> out;
  std::ifstream f(path, std::ios::binary);
  uint32_t n;
  while (f.read(reinterpret_cast<char*>(&n), 4)) {
    std::string s(n, '\0');
    if (n) f.read(&s[0], n);
    out.push_back(std::move(s));
  }
  return out;
}
static void print_hex(const std::string& s) {
  for (unsigned char c : s) printf("%02x", c);
}
static void print_ids(const char* tag, const std::vector<int32_t>& ids) {
  printf("%s %zu", tag, ids.size());
  for (int32_t v : ids) printf(" %d", v);
  printf("\n");
}

// every Tokenizer method the service reaches, through the abstract base (tokenizer.h:28-46)
static int drive_tokenizer(const Tokenizer& tok, const std::vector<std::string>& cases) {
  printf("vocab %zu\n", tok.vocab_size());
  std::unique_ptr<Tokenizer> clone = tok.clone();   // scheduler.cpp:274-277: one clone per worker thread
  for (const std::string& text : cases) {
    std::vector<int32_t> ids, ids2;
    if (!tok.encode(text, &ids)) { printf("ids FAIL\n"); continue; }
    print_ids("ids", ids);
    if (!clone->encode(text, &ids2) || ids2 != ids) { printf("clone mismatch\n"); return 1; }
    printf("dec ");
    print_hex(tok.decode(Slice<int32_t>(ids.data(), ids.size()), /*skip_special_tokens=*/false));
    printf("\n");
    if (!ids.empty()) {
      const std::string piece = tok.id_to_token(ids[0]);
      auto back = tok.token_to_id(piece);
      printf("tok %d ", back.has_value() ? *back : -1);
      print_hex(piece);
      printf("\n");
    }
  }
  printf("unknown %d\n", tok.token_to_id("\x01 no such token \x02").has_value() ? 1 : 0);
  return 0;
}

// a stock tokenizer stand-in that records what it was asked to do
class CountingTokenizer final : public Tokenizer {
 public:
  explicit CountingTokenizer(int* calls) : calls_(calls) {}
  bool encode(const std::string_view& text, std::vector<int32_t>* ids) const override {
    ++*calls_;
    for (unsigned char c : text) ids->push_back(1000000 + c);   // recognisable ids
    return true;
  }
  std::string decode(const Slice<int32_t>&, bool) const override { return ""; }
  std::optional<int32_t> token_to_id(const std::string_view&) const override { return std::nullopt; }
  std::string id_to_token(int32_t) const override { return ""; }
  size_t vocab_size() const override { return 1; }
  std::unique_ptr<Tokenizer> clone() const override { return std::make_unique<CountingTokenizer>(calls_); }
 private:
  int* calls_;
};

static int run_route(uint64_t seed) {
  std::mt19937_64 rng(seed);
  const int n_inst = 48;
  std::vector<std::string> names;
  for (int i = 0; i < n_inst; ++i) names.push_back("10.0." + std::to_string(i / 8) + "." + std::to_string(i % 8) + ":9000");
  // reference side
  FLAGS_xxh3_128bits_seed = 1024;
  auto etcd = std::make_shared<EtcdClient>("fake://seams", "");
  Options opt;
  opt.block_size(128);
  auto ref_mgr = std::make_shared<GlobalKVCacheMgr>(opt, etcd, true);
  auto ref_inst = std::make_shared<InstanceMgr>();
  CacheAwareRouting ref_car(ref_inst, ref_mgr);
  // GPU side
  xllm_ingest_config cfg{};
  cfg.block_size = 128;
  cfg.xxh3_seed = 1024;
  cfg.index_capacity = 1 << 16;
  xllm_ingest_t h = nullptr;
  if (xllm_ingest_create(&cfg, &h) != XLLM_OK) { printf("create: %s\n", xllm_last_error()); return 1; }
  auto index = std::make_shared<GpuGlobalKVCacheIndex>(h);
  GpuCacheAwareRouting car(ref_inst, index, 128);
  LoadBalancePolicy* policy = &car;   // the seam Scheduler holds (scheduler.h: unique_ptr<LoadBalancePolicy>)

  std::vector<std::vector<int32_t>> prompts;
  for (int p = 0; p < 6; ++p) {
    std::vector<int32_t> t(128 * (4 + p * 9));
    for (auto& v : t) v = (int32_t)(rng() % 150000);
    prompts.push_back(t);
  }
  auto keys_of = [&](const std::vector<int32_t>& t) {
    std::vector<std::string> ks;
    uint8_t k[16];
    for (size_t b = 0; b + 128 <= t.size(); b += 128) {
      xxh3_128bits_hash(b ? k : nullptr, Slice<int32_t>(t.data() + b, 128), k);   // the reference's own hash
      ks.emplace_back(reinterpret_cast<const char*>(k), 16);
    }
    return ks;
  };
  std::vector<std::vector<std::string>> pkeys;
  for (auto& p : prompts) pkeys.push_back(keys_of(p));

  int checked = 0, routed = 0, mismatched = 0;
  for (int round = 0; round < 10; ++round) {
    // instance view
    for (int i = 0; i < n_inst; ++i) {
      if (rng() % 4 == 0 && round) continue;
      const InstanceType type = (InstanceType)(rng() % 4);
      const bool sched = rng() % 10 != 0;
      InstanceMetaInfo info(names[i], "rpc", type);
      info.runtime_state = sched ? InstanceRuntimeState::ACTIVE : InstanceRuntimeState::SUSPECT;
      ref_inst->instances_[names[i]] = info;
      index->set_instance(names[i], type, sched);
      // distinct usages: the reference breaks ties by unordered_map order, the device by lowest id
      LoadMetrics lm(rng() % 7, (float)((i * 37 + round * 11) % 997) / 1000.0f);
      ref_inst->load_metrics_[names[i]] = lm;
      index->set_load_metrics(names[i], lm);
    }
    // KvCacheEvents
    for (int e = 0; e < 40; ++e) {
      const std::string& name = names[rng() % n_inst];
      const auto& ks = pkeys[rng() % pkeys.size()];
      proto::KvCacheEvent ev;
      const size_t upto = 1 + rng() % ks.size();
      if (rng() % 3) for (size_t i = 0; i < upto; ++i) ev.add_stored_cache(ks[i]);
      // offloads (HBM -> DRAM -> SSD) only on the first half of a prompt's blocks, which the anchor instance below
      // re-stores every window: the reference's match dereferences an empty hbm set for a block held only in
      // DRAM / SSD (global_kvcache_mgr.cpp:113-114,123-124), so every matched block keeps an HBM holder here
      if (rng() % 2 == 0 && name != names[0])
        for (int k = 0; k < 3; ++k) ev.add_offload_cache(ks[rng() % (ks.size() / 2)]);
      if (rng() % 5 == 0) ev.add_removed_cache(ks[rng() % ks.size()]);
      ref_mgr->record_updated_kvcaches(name, ev);
      index->record_updated_kvcaches(name, ev);
    }
    // one anchor instance stores everything so no matched block is ever without an HBM holder
    {
      proto::KvCacheEvent ev;
      for (auto& ks : pkeys) for (size_t i = 0; i < ks.size() / 2; ++i) ev.add_stored_cache(ks[i]);
      ref_mgr->record_updated_kvcaches(names[0], ev);
      index->record_updated_kvcaches(names[0], ev);
    }
    ref_mgr->upload_kvcache();
    if (!index->upload_kvcache()) { printf("publish: %s\n", xllm_last_error()); return 1; }
    // requests
    for (int q = 0; q < 60; ++q) {
      const auto& base = prompts[rng() % prompts.size()];
      auto req_a = std::make_shared<Request>(), req_b = std::make_shared<Request>();
      std::vector<int32_t> t(base.begin(), base.begin() + (rng() % (base.size() + 1)));
      for (int extra = (int)(rng() % 300); extra > 0; --extra) t.push_back((int32_t)(rng() % 150000));
      req_a->token_ids = t;
      req_b->token_ids = t;
      const bool ok_ref = ref_car.select_instances_pair(req_a);
      const bool ok_gpu = policy->select_instances_pair(req_b);
      OverlapScores os_ref, os_gpu;
      ref_mgr->match(Slice<int32_t>(t.data(), t.size()), &os_ref);
      index->match(Slice<int32_t>(t.data(), t.size()), 128, &os_gpu);
      ++checked;
      if (ok_ref != ok_gpu || os_ref.max_block_num != os_gpu.max_block_num ||
          os_ref.max_matched_block_num != os_gpu.max_matched_block_num || os_ref.instances != os_gpu.instances ||
          os_ref.hbm_instance_score != os_gpu.hbm_instance_score ||
          os_ref.dram_instance_score != os_gpu.dram_instance_score ||
          os_ref.ssd_instance_score != os_gpu.ssd_instance_score) {
        ++mismatched;
        printf("MISMATCH match round %d q %d\n", round, q);
        continue;
      }
      if (ok_ref) {
        ++routed;
        if (req_a->routing.prefill_name != req_b->routing.prefill_name ||
            req_a->routing.decode_name != req_b->routing.decode_name) {
          ++mismatched;
          printf("MISMATCH routing round %d q %d: ref %s / %s, gpu %s / %s\n", round, q,
                 req_a->routing.prefill_name.c_str(), req_a->routing.decode_name.c_str(),
                 req_b->routing.prefill_name.c_str(), req_b->routing.decode_name.c_str());
        }
      }
    }
  }
  // an instance leaves; its id is recycled for a newcomer; a 65th distinct name is refused, not fatal
  index->release_instance(names[1]);
  const int recycled = index->instance_id("newcomer:1");
  for (int i = 0; i < 80; ++i) index->instance_id("overflow-" + std::to_string(i));
  printf("route checked %d routed %d mismatched %d recycled_id %d overflow_id %d\n", checked, routed, mismatched,
         recycled, index->instance_id("overflow-79"));
  index.reset();
  xllm_ingest_destroy(h);
  return mismatched != 0;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string mode = argv[1];
  int rc = 2;
  if (mode == "fast" && argc >= 4) {
    FastTokenizer tok(argv[2]);   // CHECK-fails (aborts) when the library refuses the model: fast_tokenizer.cpp:10-11
    rc = drive_tokenizer(tok, read_cases(argv[3]));
  } else if (mode == "gpu" && argc >= 4) {
    int calls = 0;
    GpuTokenizer tok(argv[2], 0, 128, 1024, std::make_unique<CountingTokenizer>(&calls));
    rc = drive_tokenizer(tok, read_cases(argv[3]));
    printf("delegated %d\n", calls);
  } else if (mode == "route") {
    rc = run_route(argc >= 3 ? strtoull(argv[2], nullptr, 10) : 1);
  }
  printf(rc == 0 ? "OK\n" : "FAILED\n");
  return rc;
}
