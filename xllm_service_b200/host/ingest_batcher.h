// ingest_batcher.h — host-side micro-batching layer in front of xllm_ingest_batch.
//
// The reference runs the ingest path synchronously, one request per brpc worker thread
// (xllm_service/http_service/service.cpp:396,474 -> Scheduler::schedule, scheduler.cpp:107-153; up to 32
// workers / 128 concurrent requests, global_gflags.cpp:32-36).  A GPU wants thousands of requests
// per launch, so worker threads hand their request to this batcher and block until the batch that
// carries it has gone through the device: the call stays "one request in -> ids + routing out"
// (SURVEY.md §8f rank 2).  Header-only, depends only on the C-ABI.
//
// Policy: the first thread of a batch becomes its leader; it collects requests for at least `max_wait_us` and for as
// long as the device is still busy with an earlier batch (closing early would only queue a small batch behind it),
// or until `max_batch` requests / `max_bytes` text bytes are queued; then it copies the prompts into one of TWO
// page-locked staging sets, runs ONE xllm_ingest_batch (device calls are serialised), hands the results out and
// wakes its followers.  The next batch assembles meanwhile, and batch k+1 can be on the device while the results
// of batch k are still being handed out.
//
// Online / offline mix (BASELINE config 5; Request::offline, request/request.h:41 — "preemptive execution for online
// requests and best-effort execution for offline requests", README.md:40): submit(prompt, out, /*offline=*/true) parks
// the request in a deferred queue instead of opening or extending a batch.  Whenever a batch of online requests
// closes, the room it has left (requests and bytes) is filled with deferred offline requests, oldest first, so they
// ride along for free and never delay an online request; an offline request nobody picked up within
// `offline_defer_us` stops waiting and goes through the online path itself (no starvation when there is no online
// traffic).
#pragma once
#include <stdint.h>
#include <string.h>

#include <chrono>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <string_view>
#include <vector>

#include "xllm_ingest.h"

// Weak: a program that links the batcher against an older build of the library (or a stand-in for the C-ABI without
// this entry point) still links; the handle then keeps its default NFC policy.
extern "C" int xllm_set_nfc_policy(xllm_ingest_t h, int32_t policy) __attribute__((weak));

namespace xllm_host {

struct IngestResult {
  int32_t status = XLLM_ERR_CUDA;     // 0 ok, XLLM_ENC_TRUNCATED, or a negative XLLM_ERR_*
  std::vector<int32_t> token_ids;     // Request::token_ids (request/request.h)
  xllm_routing_out routing{};         // Request::routing as instance ids
  xllm_match_out match{};             // OverlapScores
};

class IngestBatcher {
 public:
  // `h` must outlive the batcher.  max_tokens bounds the ids returned per request.
  IngestBatcher(xllm_ingest_t h, int max_batch, size_t max_bytes, int max_tokens, int block_size, int max_wait_us,
                bool want_routing, int offline_defer_us = 20000, int64_t memo_persist_requests = 1 << 20)
      : h_(h), max_batch_(max_batch), max_bytes_(max_bytes), max_tokens_(max_tokens),
        keys_stride_(max_tokens / block_size), max_wait_us_(max_wait_us), want_routing_(want_routing),
        offline_defer_us_(offline_defer_us) {
    ok_ = true;
    // a service's batches are small and come one after the other: keep the tokenizer's word memo across launches
    // (cleared every memo_persist_requests requests) instead of starting every batch from an empty table
    xllm_set_memo_policy(h, memo_persist_requests);
    // tokenizers with `normalizer: NFC` (Qwen2 family): accept every request that is in NFC, not only those made of
    // NFC-inert chars, so text with combining marks (Thai, Devanagari, ...) stays on the device
    if (xllm_set_nfc_policy) xllm_set_nfc_policy(h, XLLM_NFC_VERIFY);
    // vocabularies below 65 536 pieces: take the ids as uint16 (half the bytes over PCIe) and widen them in hand_out,
    // during the copy into the caller's std::vector<int32_t> that happens anyway
    int32_t vocab = 0;
    narrow_ids_ = xllm_vocab_size(h, &vocab) == XLLM_OK && vocab > 0 && vocab < 65536;
    for (Staging& s : sets_) {
      ok_ = ok_ && xllm_host_alloc(reinterpret_cast<void**>(&s.text), max_bytes) == XLLM_OK &&
            xllm_host_alloc(reinterpret_cast<void**>(&s.offsets), sizeof(int64_t) * (max_batch + 1)) == XLLM_OK &&
            xllm_host_alloc(reinterpret_cast<void**>(&s.ids), (narrow_ids_ ? sizeof(uint16_t) : sizeof(int32_t)) *
                                                                   (size_t)max_batch * max_tokens) == XLLM_OK &&
            xllm_host_alloc(reinterpret_cast<void**>(&s.n_ids), sizeof(int32_t) * max_batch) == XLLM_OK &&
            xllm_host_alloc(reinterpret_cast<void**>(&s.status), sizeof(int32_t) * max_batch) == XLLM_OK &&
            xllm_host_alloc(reinterpret_cast<void**>(&s.match), sizeof(xllm_match_out) * max_batch) == XLLM_OK &&
            xllm_host_alloc(reinterpret_cast<void**>(&s.routing), sizeof(xllm_routing_out) * max_batch) == XLLM_OK;
    }
    free_sets_ = {0, 1};
  }
  ~IngestBatcher() {
    for (Staging& s : sets_) {
      xllm_host_free(s.text); xllm_host_free(s.offsets); xllm_host_free(s.ids); xllm_host_free(s.n_ids);
      xllm_host_free(s.status); xllm_host_free(s.match); xllm_host_free(s.routing);
    }
  }
  bool ok() const { return ok_; }
  uint64_t batches() const { return n_batches_; }
  uint64_t requests() const { return n_requests_; }
  uint64_t offline_piggybacked() const { return n_piggyback_; }   // offline requests that rode in an online batch

  // Blocks until the request has been tokenised (+ matched and routed).  Thread-safe.  offline = best effort: see
  // the header comment.
  void submit(std::string_view prompt, IngestResult* out, bool offline = false) {
    std::unique_lock<std::mutex> lk(mu_);
    if (!ok_ || prompt.size() > max_bytes_) { out->status = XLLM_ERR_CAPACITY; return; }
    if (offline && offline_defer_us_ > 0) {
      auto d = std::make_shared<Deferred>();
      d->item = Item{prompt, out};
      deferred_.push_back(d);
      const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(offline_defer_us_);
      cv_done_.wait_until(lk, deadline, [&] { return d->batch != nullptr; });
      if (d->batch) {   // an online batch took it along
        std::shared_ptr<Batch> b = d->batch;
        cv_done_.wait(lk, [&] { return b->done; });
        return;
      }
      for (auto it = deferred_.begin(); it != deferred_.end(); ++it)   // nobody came: go through the front door
        if (*it == d) { deferred_.erase(it); break; }
    }
    // wait for room in the batch that is being assembled
    cv_room_.wait(lk, [&] {
      return !cur_ || ((int)cur_->items.size() < max_batch_ && bytes_ + prompt.size() <= max_bytes_);
    });
    if (!cur_) { cur_ = std::make_shared<Batch>(); bytes_ = 0; }
    std::shared_ptr<Batch> b = cur_;
    b->items.push_back(Item{prompt, out});
    bytes_ += prompt.size();
    if (b->items.size() > 1) {  // follower
      if ((int)b->items.size() >= max_batch_ || bytes_ >= max_bytes_) cv_full_.notify_all();
      cv_done_.wait(lk, [&] { return b->done; });
      return;
    }
    // leader: give followers max_wait_us to join — and as long as the device is busy anyway — or go when full
    auto full = [&] { return (int)b->items.size() >= max_batch_ || bytes_ >= max_bytes_; };
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(max_wait_us_);
    cv_full_.wait_until(lk, deadline, full);
    cv_full_.wait(lk, [&] { return full() || (!dev_busy_ && !free_sets_.empty()); });
    // closing: deferred offline requests fill whatever room is left, oldest first
    while (!deferred_.empty() && (int)b->items.size() < max_batch_ &&
           bytes_ + deferred_.front()->item.prompt.size() <= max_bytes_) {
      std::shared_ptr<Deferred> d = deferred_.front();
      deferred_.pop_front();
      b->items.push_back(d->item);
      bytes_ += d->item.prompt.size();
      d->batch = b;
      ++n_piggyback_;
    }
    cv_done_.notify_all();   // the riders stop watching their deadline
    cur_.reset();  // closed: the next batch starts assembling now
    bytes_ = 0;
    cv_room_.notify_all();
    cv_set_.wait(lk, [&] { return !dev_busy_ && !free_sets_.empty(); });
    const int set = free_sets_.back();
    free_sets_.pop_back();
    dev_busy_ = true;
    lk.unlock();
    const int rc = device_call(*b, sets_[set]);
    lk.lock();
    dev_busy_ = false;  // the next batch may close and go while this one's results are handed out
    cv_full_.notify_all();
    cv_set_.notify_all();
    lk.unlock();
    hand_out(*b, sets_[set], rc);
    lk.lock();
    free_sets_.push_back(set);
    b->done = true;
    ++n_batches_;
    n_requests_ += (uint64_t)b->items.size();
    cv_done_.notify_all();
    cv_full_.notify_all();
    cv_set_.notify_all();
  }

 private:
  struct Item {
    std::string_view prompt;
    IngestResult* out;
  };
  struct Batch {
    std::vector<Item> items;
    bool done = false;
  };
  struct Deferred {   // an offline request waiting for a ride
    Item item;
    std::shared_ptr<Batch> batch;   // set when an online batch took it
  };
  struct Staging {  // page-locked buffers of one batch in flight
    uint8_t* text = nullptr;
    int64_t* offsets = nullptr;
    int32_t* ids = nullptr;
    int32_t* n_ids = nullptr;
    int32_t* status = nullptr;
    xllm_match_out* match = nullptr;
    xllm_routing_out* routing = nullptr;
  };
  // copy in + one device call, without the batcher lock (the callers of this batch are all blocked)
  int device_call(Batch& batch, Staging& s) {
    const int n = (int)batch.items.size();
    int64_t at = 0;
    for (int i = 0; i < n; ++i) {
      s.offsets[i] = at;
      memcpy(s.text + at, batch.items[i].prompt.data(), batch.items[i].prompt.size());
      at += (int64_t)batch.items[i].prompt.size();
    }
    s.offsets[n] = at;
    xllm_ingest_io io;
    memset(&io, 0, sizeof(io));
    io.n_req = n;
    io.text = s.text;
    io.offsets = s.offsets;
    if (narrow_ids_) io.ids_u16 = reinterpret_cast<uint16_t*>(s.ids);
    else io.ids = s.ids;
    io.ids_stride = max_tokens_;
    io.n_ids = s.n_ids;
    io.status = s.status;
    io.match = want_routing_ ? s.match : nullptr;
    io.routing = want_routing_ ? s.routing : nullptr;
    std::lock_guard<std::mutex> dev(dev_mu_);  // one launch at a time per handle (dev_busy_ already ensures it)
    return xllm_ingest_batch(h_, &io);
  }
  void hand_out(Batch& batch, Staging& s, int rc) {
    const int n = (int)batch.items.size();
    for (int i = 0; i < n; ++i) {
      IngestResult* o = batch.items[i].out;
      o->status = rc != XLLM_OK ? rc : s.status[i];
      if (rc == XLLM_OK && s.status[i] >= 0) {
        const int32_t keep = s.n_ids[i] < max_tokens_ ? s.n_ids[i] : max_tokens_;
        if (narrow_ids_) {
          const uint16_t* row = reinterpret_cast<const uint16_t*>(s.ids) + (size_t)i * max_tokens_;
          o->token_ids.assign(row, row + keep);   // widens uint16 -> int32
        } else {
          o->token_ids.assign(s.ids + (size_t)i * max_tokens_, s.ids + (size_t)i * max_tokens_ + keep);
        }
        if (want_routing_) { o->match = s.match[i]; o->routing = s.routing[i]; }
      }
    }
  }

  xllm_ingest_t h_;
  const int max_batch_;
  const size_t max_bytes_;
  const int max_tokens_;
  const int keys_stride_;
  const int max_wait_us_;
  const bool want_routing_;
  const int offline_defer_us_;
  bool narrow_ids_ = false;
  std::deque<std::shared_ptr<Deferred>> deferred_;
  uint64_t n_piggyback_ = 0;
  bool ok_ = false;
  Staging sets_[2];
  std::vector<int> free_sets_;
  std::mutex mu_, dev_mu_;
  std::condition_variable cv_room_, cv_full_, cv_done_, cv_set_;
  bool dev_busy_ = false;       // a batch is between copy-in and the return of its device call
  std::shared_ptr<Batch> cur_;  // the batch being assembled (null: none)
  size_t bytes_ = 0;            // text bytes queued in cur_
  uint64_t n_batches_ = 0, n_requests_ = 0;
};

}  // namespace xllm_host
