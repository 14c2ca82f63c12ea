// pipeline.cu — the whole ingest hot path for a batch of requests behind one C-ABI call:
//   host text -> [H2D] -> tokenize -> block-hash chain -> index probe -> match scan + routing -> [D2H]
// i.e. what Scheduler::schedule does per request between scheduler.cpp:128 and :135
// (Tokenizer::encode, then CacheAwareRouting::select_instances_pair -> GlobalKVCacheMgr::match ->
// cost_function), batched.  The batch is cut into chunks that flow through an upload, a kernel and a download
// stream so the PCIe copies of one chunk overlap the kernels of another; the caller's buffers should be
// page-locked (xllm_host_alloc: also NUMA-local to the GPU) for the copies to be asynchronous.
#include <ctype.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "../../include/xllm_ingest.h"
#include <chrono>
#include <vector>

#include "handle.h"
#include "pipeline_schedule.h"

namespace xllm {

namespace {

// Row descriptors for the hash / match stages of one chunk (request-local indices).
__global__ void prep_rows_kernel(const int32_t* __restrict__ n_ids, int n, int64_t ids_stride, int64_t keys_stride,
                                 int block_size, int64_t* __restrict__ tok_start, int32_t* __restrict__ n_tok,
                                 int64_t* __restrict__ key_start, int32_t* __restrict__ n_blocks) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  int64_t t = n_ids[r];
  if (t > ids_stride) t = ids_stride;  // truncated rows hash what was written
  int64_t nb = t / block_size;
  if (nb > keys_stride) nb = keys_stride;
  tok_start[r] = (int64_t)r * ids_stride;
  n_tok[r] = (int32_t)(nb * block_size);
  key_start[r] = (int64_t)r * keys_stride;
  n_blocks[r] = (int32_t)nb;
}

// Narrow download (xllm_ingest_io::ids_u16): int32 ids -> uint16, 8 ids per thread (rows are 16-byte aligned when
// ids_stride is a multiple of 8; the tail of an odd-sized buffer goes one id at a time).
__global__ void narrow_ids_kernel(const int32_t* __restrict__ ids, uint16_t* __restrict__ out, size_t n) {
  const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const int4 a = *reinterpret_cast<const int4*>(ids + i), b = *reinterpret_cast<const int4*>(ids + i + 4);
    uint4 o;
    o.x = (uint32_t)(uint16_t)a.x | ((uint32_t)(uint16_t)a.y << 16);
    o.y = (uint32_t)(uint16_t)a.z | ((uint32_t)(uint16_t)a.w << 16);
    o.z = (uint32_t)(uint16_t)b.x | ((uint32_t)(uint16_t)b.y << 16);
    o.w = (uint32_t)(uint16_t)b.z | ((uint32_t)(uint16_t)b.w << 16);
    *reinterpret_cast<uint4*>(out + i) = o;
  } else {
    for (size_t k = i; k < n; ++k) out[k] = (uint16_t)ids[k];
  }
}

// Segmented requests: one warp per request walks its segments in order and splices the ids of encoded text pieces
// (ragged temporary rows) and of ready-made id spans into the request's row.  n_ids = the full count even when it
// exceeds the row; status = the first failing piece's code, else truncated / ok.
__global__ void __launch_bounds__(128) assemble_segments_kernel(
    const int32_t* __restrict__ req_seg, const int32_t* __restrict__ seg_len, const int64_t* __restrict__ seg_src,
    const int32_t* __restrict__ piece_ids, const int64_t* __restrict__ piece_out_start,
    const int32_t* __restrict__ piece_out_cap, const int32_t* __restrict__ piece_n,
    const int32_t* __restrict__ piece_status, const int32_t* __restrict__ span, int m, int32_t* __restrict__ ids,
    int64_t ids_stride, int32_t* __restrict__ n_ids, int32_t* __restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= m) return;
  int32_t* row = ids + (int64_t)r * ids_stride;
  int64_t at = 0;
  int32_t st = 0;
  for (int s = req_seg[r]; s < req_seg[r + 1]; ++s) {
    const int32_t len = seg_len[s];
    const int32_t* src;
    int64_t n, have;
    if (len < 0) {   // a text piece
      const int64_t p = seg_src[s];
      int32_t ps = piece_status[p];
      n = piece_n[p];
      // a piece whose ids outgrew its temporary row (a normaliser expansion of more than one id per input byte, e.g.
      // U+FDFA): the row holds only a prefix, so the request fails loudly instead of being spliced with a hole
      if (ps >= 0 && n > piece_out_cap[p]) ps = XLLM_ERR_CAPACITY;
      if (ps < 0 && st >= 0) st = ps;
      have = n < piece_out_cap[p] ? n : piece_out_cap[p];   // ids actually present in the temporary row
      src = piece_ids + piece_out_start[p];
      if (ps < 0) { n = 0; have = 0; }
    } else {
      n = have = len;
      src = span + seg_src[s];
    }
    int64_t room = ids_stride - at;
    if (room < 0) room = 0;
    const int64_t copy = have < room ? have : room;
    for (int64_t i = lane; i < copy; i += 32) row[at + i] = src[i];
    at += n;
  }
  if (lane == 0) {
    n_ids[r] = st < 0 ? 0 : (int32_t)at;
    status[r] = st < 0 ? st : (at > ids_stride ? 1 : 0);
  }
}

// Sharded index: the exchange runs once per batch, so every chunk also files its rows in batch-wide descriptors.
__global__ void batch_rows_kernel(const int32_t* __restrict__ chunk_n_blocks, int m, int64_t row0, int64_t keys_stride,
                                  int64_t* __restrict__ all_key_start, int32_t* __restrict__ all_n_blocks) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  all_key_start[row0 + r] = (row0 + r) * keys_stride;
  all_n_blocks[row0 + r] = chunk_n_blocks[r];
}

}  // namespace

// n: rows of the offsets table (requests, or text pieces of segmented requests); n_req: request rows of the outputs
int PipeSlot::ensure(size_t text_bytes, int n, int64_t ids_stride, int64_t keys_stride, int n_req) {
  int rc;
  if (n_req < 0) n_req = n;
  if ((rc = d_text.reserve(text_bytes + 64)) != XLLM_OK) return rc;
  if ((rc = d_offsets.reserve((size_t)(n + 1) * 8)) != XLLM_OK) return rc;
  if ((rc = d_ids.reserve((size_t)n_req * (size_t)ids_stride * 4 + 64)) != XLLM_OK) return rc;
  if ((rc = d_n_ids.reserve((size_t)n * 4)) != XLLM_OK) return rc;
  if ((rc = d_status.reserve((size_t)n * 4)) != XLLM_OK) return rc;
  if ((rc = d_tok_start.reserve((size_t)n * 8)) != XLLM_OK) return rc;
  if ((rc = d_n_tok.reserve((size_t)n * 4)) != XLLM_OK) return rc;
  if ((rc = d_key_start.reserve((size_t)n * 8)) != XLLM_OK) return rc;
  if ((rc = d_n_blocks.reserve((size_t)n * 4)) != XLLM_OK) return rc;
  if ((rc = d_keys.reserve((size_t)n_req * (size_t)keys_stride * 16 + 64)) != XLLM_OK) return rc;
  if ((rc = d_match.reserve((size_t)n * sizeof(MatchOut))) != XLLM_OK) return rc;
  if ((rc = d_routing.reserve((size_t)n * sizeof(RoutingOut))) != XLLM_OK) return rc;
  return XLLM_OK;
}

void PipeSlot::release() {
  d_defer.release();
  d_memo.release();
  d_text.release(); d_offsets.release(); d_ids.release(); d_n_ids.release(); d_status.release();
  d_tok_start.release(); d_n_tok.release(); d_key_start.release(); d_n_blocks.release();
  d_keys.release(); d_masks.release(); d_match.release(); d_routing.release();
  d_ids16.release();
  d_piece_ids.release(); d_piece_n.release(); d_piece_status.release(); d_piece_out_start.release();
  d_piece_out_cap.release(); d_seg_len.release(); d_seg_src.release(); d_req_seg.release(); d_span.release();
  for (int k = 0; k < 3; ++k) {
    if (ev[k]) cudaEventDestroy(ev[k]);
    ev[k] = nullptr;
  }
  if (counters) cudaFree(counters);
  counters = nullptr;
  busy = false;
}

}  // namespace xllm

using namespace xllm;

extern "C" {

// CPUs local to the current device's PCIe root (sysfs local_cpulist, e.g. "0-31,64-95")
static bool gpu_local_cpus(cpu_set_t* set) {
  int dev = 0;
  char bus[32] = {0};
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetPCIBusId(bus, (int)sizeof(bus), dev) != cudaSuccess) return false;
  for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
  char path[128];
  snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/local_cpulist", bus);
  FILE* f = fopen(path, "r");
  if (!f) return false;
  char line[512] = {0};
  const bool got = fgets(line, sizeof(line), f) != nullptr;
  fclose(f);
  if (!got) return false;
  CPU_ZERO(set);
  int n = 0;
  for (char* p = line; *p && *p != '\n';) {
    char* end;
    const long a = strtol(p, &end, 10);
    if (end == p) break;
    long b = a;
    p = end;
    if (*p == '-') { b = strtol(p + 1, &end, 10); p = end; }
    for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int)c, set); ++n; }
    if (*p == ',') ++p;
  }
  return n > 0;
}

int xllm_host_alloc(void** out, size_t bytes) {
  if (!out) return XLLM_ERR_INVALID_ARG;
  *out = nullptr;
  // Page-locking populates the pages, on the NUMA node of the calling thread: run the allocation on a CPU next to
  // the GPU so the DMA does not cross the socket interconnect (it costs PCIe bandwidth when both directions are busy)
  cpu_set_t old_set, local_set, both;
  bool bound = false;
  if (sched_getaffinity(0, sizeof(old_set), &old_set) == 0 && gpu_local_cpus(&local_set)) {
    CPU_AND(&both, &old_set, &local_set);
    if (CPU_COUNT(&both) > 0 && sched_setaffinity(0, sizeof(both), &both) == 0) bound = true;
  }
  cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault);
  if (bound) sched_setaffinity(0, sizeof(old_set), &old_set);
  if (e != cudaSuccess) {
    set_last_error("cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return XLLM_ERR_NOMEM;
  }
  return XLLM_OK;
}
void xllm_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

static int ingest_core(xllm_ingest_t h, const xllm_ingest_io* io, const xllm_segments* seg);
int xllm_ingest_batch(xllm_ingest_t h, const xllm_ingest_io* io) { return ingest_core(h, io, nullptr); }
int xllm_ingest_batch_segments(xllm_ingest_t h, const xllm_ingest_io* io, const xllm_segments* seg) {
  if (!seg) {
    set_last_error("xllm_ingest_batch_segments: null segment table");
    return XLLM_ERR_INVALID_ARG;
  }
  return ingest_core(h, io, seg);
}

static int ingest_core(xllm_ingest_t h, const xllm_ingest_io* io, const xllm_segments* seg) {
  if (!h || !io || io->n_req < 0) {
    set_last_error("xllm_ingest_batch: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  const int32_t n = io->n_req;
  if (n == 0) return XLLM_OK;
  if (!io->offsets || !io->n_ids || !io->status || io->ids_stride <= 0 || (!io->ids && !io->ids_u16) ||
      io->keys_stride < 0 || (io->keys_stride > 0 && !io->keys)) {
    set_last_error("xllm_ingest_batch: missing buffer");
    return XLLM_ERR_INVALID_ARG;
  }
  if (!h->sp_dev) {
    set_last_error("handle has no tokenizer (tokenizer_path was not set)");
    return XLLM_ERR_UNSUPPORTED;
  }
  if (io->ids_u16 && h->sp_dev->dev().n_pieces > 65535u) {
    set_last_error("ids_u16 needs a vocabulary below 65536 pieces (this one has %u)", h->sp_dev->dev().n_pieces);
    return XLLM_ERR_UNSUPPORTED;
  }
  const bool want_match = io->match != nullptr || io->routing != nullptr;
  if (want_match && (!h->index || !h->index->ready())) {
    set_last_error("match/routing requested but the prefix index is not configured (index_capacity == 0)");
    return XLLM_ERR_UNSUPPORTED;
  }
  const int64_t keys_stride = io->keys_stride > 0 ? io->keys_stride : (want_match ? io->ids_stride / h->block_size : 0);
  // xllm_match_out keeps scores as uint16 (1 + the last matched block index, shard tuples carry the block index in 16
  // bits too): a row of more than 65 535 blocks would wrap and report an instance holding every block as absent
  const int64_t max_row_blocks = std::min(keys_stride, io->ids_stride / h->block_size);
  if (want_match && max_row_blocks > 65535) {
    set_last_error("xllm_ingest_batch: match / routing of rows of up to %lld blocks requested, the limit is 65535 "
                   "(ids_stride %lld, keys_stride %lld, block_size %d)", (long long)max_row_blocks,
                   (long long)io->ids_stride, (long long)io->keys_stride, h->block_size);
    return XLLM_ERR_INVALID_ARG;
  }
  // ---- segmented requests: where each request's text pieces and id spans start (host prefix sums)
  int64_t n_pieces = n;                    // rows of io->offsets: requests, or text pieces
  std::vector<int64_t> piece_of_req, span_of_req, seg_src;   // [n + 1], [n + 1], [n_segments]
  if (seg) {
    if (seg->n_segments < 0 || seg->n_span_ids < 0 || !seg->req_seg_start || (seg->n_segments > 0 && !seg->seg_len) ||
        (seg->n_span_ids > 0 && !seg->span_ids) || seg->req_seg_start[0] != 0 ||
        seg->req_seg_start[n] != seg->n_segments) {
      set_last_error("xllm_ingest_batch_segments: inconsistent segment table");
      return XLLM_ERR_INVALID_ARG;
    }
    piece_of_req.assign((size_t)n + 1, 0);
    span_of_req.assign((size_t)n + 1, 0);
    seg_src.assign((size_t)seg->n_segments, 0);
    int64_t pieces = 0, spans = 0;
    for (int32_t r = 0; r < n; ++r) {
      piece_of_req[(size_t)r] = pieces;
      span_of_req[(size_t)r] = spans;
      if (seg->req_seg_start[r + 1] < seg->req_seg_start[r]) {
        set_last_error("xllm_ingest_batch_segments: req_seg_start not ascending at request %d", r);
        return XLLM_ERR_INVALID_ARG;
      }
      for (int32_t s2 = seg->req_seg_start[r]; s2 < seg->req_seg_start[r + 1]; ++s2) {
        const int32_t len = seg->seg_len[s2];
        if (len < 0) seg_src[(size_t)s2] = pieces++;
        else { seg_src[(size_t)s2] = spans; spans += len; }
      }
    }
    piece_of_req[(size_t)n] = pieces;
    span_of_req[(size_t)n] = spans;
    if (spans != seg->n_span_ids) {
      set_last_error("xllm_ingest_batch_segments: id segments add up to %lld ids, n_span_ids says %lld", (long long)spans,
                     (long long)seg->n_span_ids);
      return XLLM_ERR_INVALID_ARG;
    }
    n_pieces = pieces;
  }
  for (int64_t r = 0; r < n_pieces; ++r)
    if (io->offsets[r + 1] < io->offsets[r] || io->offsets[r] < 0 ||
        io->offsets[r + 1] - io->offsets[r] > 0x7fffffffLL) {
      set_last_error("xllm_ingest_batch: bad offsets at row %lld", (long long)r);
      return XLLM_ERR_INVALID_ARG;
    }
  if (io->offsets[n_pieces] > io->offsets[0] && !io->text) return XLLM_ERR_INVALID_ARG;
  const int tmpl_ids = h->sp_dev ? (int)h->sp_dev->dev().n_prefix + (int)h->sp_dev->dev().n_suffix : 0;

  std::lock_guard<std::mutex> lock(h->mu);
  XLLM_CUDA_TRY(cudaSetDevice(h->device));
  // hash-range-sharded index: the chunks tokenise and hash as usual, their keys stay resident, and ONE exchange round
  // for the whole batch follows the last chunk (collective: every rank makes this call once per batch)
  const bool sharded = want_match && h->shard != nullptr;
  if (sharded) {
    XLLM_TRY_RC(h->d_all_keys.reserve((size_t)n * (size_t)keys_stride * 16 + 64));
    XLLM_TRY_RC(h->d_all_key_start.reserve((size_t)n * 8));
    XLLM_TRY_RC(h->d_all_n_blocks.reserve((size_t)n * 4));
    XLLM_TRY_RC(h->d_all_match.reserve((size_t)n * sizeof(MatchOut)));
    XLLM_TRY_RC(h->d_all_routing.reserve((size_t)n * sizeof(RoutingOut)));
  }
  if (want_match) {
    std::lock_guard<std::mutex> l2(*h->index_mu);
    XLLM_CUDA_TRY(cudaMemcpyAsync(h->d_inst, h->inst_host.get(), sizeof(InstanceTable), cudaMemcpyHostToDevice,
                                  h->stream));
    XLLM_CUDA_TRY(cudaStreamSynchronize(h->stream));
  }
  // Three engine streams — uploads, kernels, downloads — joined by events: each hardware engine sees its work in
  // chunk order (no stream-to-queue aliasing, no kernel waiting behind its own chunk's download), and a chunk's
  // buffers (slot = chunk mod pipe_slots) are reused only after the chunk that last held them has left the
  // download engine.
  const int chunk_req = h->pipe_chunk_req;
  const int64_t chunk_bytes = h->pipe_chunk_bytes;
  const int n_slots = h->pipe_slots;
  for (int k = 0; k < 3; ++k)
    if (!h->pipe_stream[k]) XLLM_CUDA_TRY(cudaStreamCreateWithFlags(&h->pipe_stream[k], cudaStreamNonBlocking));
  cudaStream_t s_in = h->pipe_stream[0], s_k = h->pipe_stream[1], s_out = h->pipe_stream[2];
  for (int s = 0; s < n_slots; ++s) {
    PipeSlot& sl = h->pipe[s];
    if (!sl.counters) XLLM_CUDA_TRY(cudaMalloc(&sl.counters, 64));
    for (int k = 0; k < 3; ++k)
      if (!sl.ev[k]) XLLM_CUDA_TRY(cudaEventCreateWithFlags(&sl.ev[k], cudaEventDisableTiming));
    sl.busy = false;
  }
  // XLLM_PIPE_TRACE=1: per-chunk device timeline on stderr (debugging aid)
  static const bool trace = getenv("XLLM_PIPE_TRACE") != nullptr;
  struct TraceRow { int m; double host_ms; cudaEvent_t e[5]; };
  std::vector<TraceRow> rows;
  cudaEvent_t ev_begin = nullptr;
  const auto host_t0 = std::chrono::steady_clock::now();
  if (trace) { cudaEventCreate(&ev_begin); cudaEventRecord(ev_begin, s_in); }
  auto mark = [&](int k, cudaStream_t st) {
    if (!trace) return;
    cudaEventCreate(&rows.back().e[k]);
    cudaEventRecord(rows.back().e[k], st);
  };
  int slot = 0;
  int32_t c0 = 0;
  int rc = XLLM_OK;
  h->last_chunks = 0;
  h->last_launches = 0;
  ChunkSchedule sched(chunk_req);  // ramp-up, full-size bulk, quarter-size tail (pipeline_schedule.h)
  // inside the chunk loop a CUDA error must not return at once: copies into the caller's buffers may be in flight, so
  // leave the loop and synchronise the three streams first
#define PIPE_CUDA_TRY(expr)                                                                              \
  if (cudaError_t _pe = (expr); _pe != cudaSuccess) {                                                    \
    ::xllm::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_pe));       \
    rc = XLLM_ERR_CUDA;                                                                                  \
    break;                                                                                               \
  } else                                                                                                 \
    (void)0
  while (c0 < n) {
    const int64_t target = sched.next((int64_t)n - c0);
    int32_t c1 = c0;
    // first / one-past-last row of io->offsets a request range covers (requests themselves, or their text pieces)
    auto row_of = [&](int32_t r) { return seg ? piece_of_req[(size_t)r] : (int64_t)r; };
    while (c1 < n && c1 - c0 < target &&
           (c1 == c0 || io->offsets[row_of(c1 + 1)] - io->offsets[row_of(c0)] <= chunk_bytes))
      ++c1;
    const int m = c1 - c0;
    const int64_t p0 = row_of(c0), p1 = row_of(c1);
    const int mp = (int)(p1 - p0);                     // rows the encode kernel sees: m requests, or mp text pieces
    const int64_t t0 = io->offsets[p0];
    const size_t text_bytes = (size_t)(io->offsets[p1] - t0);
    PipeSlot& sl = h->pipe[slot];
    uint8_t* chunk_keys = sl.d_keys.as<uint8_t>();
    // the slot's previous chunk has been downloaded (host wait: ensure() below may reallocate its buffers)
    if (sl.busy) PIPE_CUDA_TRY(cudaEventSynchronize(sl.ev[2]));
    if ((rc = sl.ensure(text_bytes, m > mp ? m : mp, io->ids_stride, keys_stride, m)) != XLLM_OK) break;
    xllm::SpMemo memo;
    xllm::SpEncodePlan plan;
    if ((rc = encode_reserve(h, mp, &sl.d_defer, &sl.d_memo, &sl.memo_age, &memo, &plan)) != XLLM_OK) break;
    if (trace) {
      rows.push_back(TraceRow{m, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count(), {}});
      mark(0, s_in);
    }
    // ---- upload
    if (text_bytes)
      PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_text.p, io->text + t0, text_bytes, cudaMemcpyHostToDevice, s_in));
    PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_offsets.p, io->offsets + p0, (size_t)(mp + 1) * 8, cudaMemcpyHostToDevice, s_in));
    int64_t piece_ids_total = 0;
    if (seg) {
      // ragged temporary rows for the pieces: a piece of b bytes yields at most b + 1 ids (+ template ids)
      const int32_t s0 = seg->req_seg_start[c0], s1 = seg->req_seg_start[c1];
      const int64_t sp0 = span_of_req[(size_t)c0], sp1 = span_of_req[(size_t)c1];
      std::vector<int64_t>& ostart = sl.h_piece_out_start;
      std::vector<int32_t>& ocap = sl.h_piece_out_cap;
      std::vector<int32_t>& rseg = sl.h_req_seg;
      std::vector<int64_t>& ssrc = sl.h_seg_src;
      ostart.resize((size_t)mp + 1);
      ocap.resize((size_t)mp + 1);
      for (int k = 0; k < mp; ++k) {
        ostart[(size_t)k] = piece_ids_total;
        ocap[(size_t)k] = (int32_t)(io->offsets[p0 + k + 1] - io->offsets[p0 + k]) + 2 + tmpl_ids;
        piece_ids_total += ocap[(size_t)k];
      }
      rseg.resize((size_t)m + 1);
      for (int k = 0; k <= m; ++k) rseg[(size_t)k] = seg->req_seg_start[c0 + k] - s0;
      ssrc.resize((size_t)(s1 - s0) + 1);
      for (int32_t k = s0; k < s1; ++k)   // chunk-local: piece index / span offset
        ssrc[(size_t)(k - s0)] = seg_src[(size_t)k] - (seg->seg_len[k] < 0 ? p0 : sp0);
      if ((rc = sl.d_piece_ids.reserve((size_t)piece_ids_total * 4 + 64)) != XLLM_OK) break;
      if ((rc = sl.d_piece_n.reserve((size_t)mp * 4 + 4)) != XLLM_OK) break;
      if ((rc = sl.d_piece_status.reserve((size_t)mp * 4 + 4)) != XLLM_OK) break;
      if ((rc = sl.d_piece_out_start.reserve((size_t)mp * 8 + 8)) != XLLM_OK) break;
      if ((rc = sl.d_piece_out_cap.reserve((size_t)mp * 4 + 4)) != XLLM_OK) break;
      if ((rc = sl.d_seg_len.reserve((size_t)(s1 - s0) * 4 + 4)) != XLLM_OK) break;
      if ((rc = sl.d_seg_src.reserve((size_t)(s1 - s0) * 8 + 8)) != XLLM_OK) break;
      if ((rc = sl.d_req_seg.reserve((size_t)(m + 1) * 4)) != XLLM_OK) break;
      if ((rc = sl.d_span.reserve((size_t)(sp1 - sp0) * 4 + 4)) != XLLM_OK) break;
      if (mp) {
        PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_piece_out_start.p, ostart.data(), (size_t)mp * 8, cudaMemcpyHostToDevice, s_in));
        PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_piece_out_cap.p, ocap.data(), (size_t)mp * 4, cudaMemcpyHostToDevice, s_in));
      }
      if (s1 > s0) {
        PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_seg_len.p, seg->seg_len + s0, (size_t)(s1 - s0) * 4, cudaMemcpyHostToDevice, s_in));
        PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_seg_src.p, ssrc.data(), (size_t)(s1 - s0) * 8, cudaMemcpyHostToDevice, s_in));
      }
      PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_req_seg.p, rseg.data(), (size_t)(m + 1) * 4, cudaMemcpyHostToDevice, s_in));
      if (sp1 > sp0)
        PIPE_CUDA_TRY(cudaMemcpyAsync(sl.d_span.p, seg->span_ids + sp0, (size_t)(sp1 - sp0) * 4, cudaMemcpyHostToDevice, s_in));
    }
    PIPE_CUDA_TRY(cudaEventRecord(sl.ev[0], s_in));
    mark(1, s_in);
    // ---- kernels: tokenize -> row prep -> chained block hash -> index probe -> match scan + routing
    PIPE_CUDA_TRY(cudaStreamWaitEvent(s_k, sl.ev[0], 0));
    if (!seg) {
      xllm::SpLaunchOpts opts;
      opts.nfc_verify = plan.nfc_verify;
      PIPE_CUDA_TRY(sp_encode_launch(h->sp_dev->dev(), sl.d_text.as<uint8_t>() - t0, sl.d_offsets.as<int64_t>(), m,
                                     sl.d_ids.as<int32_t>(), io->ids_stride, sl.d_n_ids.as<int32_t>(),
                                     sl.d_status.as<int32_t>(), sl.counters, sl.d_defer.p, s_k, memo, opts));
    } else {
      xllm::SpLaunchOpts opts;
      opts.nfc_verify = plan.nfc_verify;
      opts.out_start = sl.d_piece_out_start.as<int64_t>();
      opts.out_cap = sl.d_piece_out_cap.as<int32_t>();
      PIPE_CUDA_TRY(sp_encode_launch(h->sp_dev->dev(), sl.d_text.as<uint8_t>() - t0, sl.d_offsets.as<int64_t>(), mp,
                                     sl.d_piece_ids.as<int32_t>(), 0, sl.d_piece_n.as<int32_t>(),
                                     sl.d_piece_status.as<int32_t>(), sl.counters, sl.d_defer.p, s_k, memo,
                                     opts));
      assemble_segments_kernel<<<(m + 3) / 4, 128, 0, s_k>>>(
          sl.d_req_seg.as<int32_t>(), sl.d_seg_len.as<int32_t>(), sl.d_seg_src.as<int64_t>(),
          sl.d_piece_ids.as<int32_t>(), sl.d_piece_out_start.as<int64_t>(), sl.d_piece_out_cap.as<int32_t>(),
          sl.d_piece_n.as<int32_t>(), sl.d_piece_status.as<int32_t>(), sl.d_span.as<int32_t>(), m,
          sl.d_ids.as<int32_t>(), io->ids_stride, sl.d_n_ids.as<int32_t>(), sl.d_status.as<int32_t>());
      PIPE_CUDA_TRY(cudaGetLastError());
      h->last_launches += 1;
    }
    mark(2, s_k);
    if (keys_stride > 0 || want_match) {
      // keys_stride == 0 with match / routing requested (ids_stride < block_size): every request has 0 blocks, the
      // match is all-zero and routing takes get_load_metrics' least-loaded fallback, as the reference does for a
      // prompt shorter than one block (global_kvcache_mgr.cpp:77-79, instance_mgr.cpp:312-358)
      prep_rows_kernel<<<(m + 127) / 128, 128, 0, s_k>>>(sl.d_n_ids.as<int32_t>(), m, io->ids_stride, keys_stride,
                                                        h->block_size, sl.d_tok_start.as<int64_t>(),
                                                        sl.d_n_tok.as<int32_t>(), sl.d_key_start.as<int64_t>(),
                                                        sl.d_n_blocks.as<int32_t>());
      PIPE_CUDA_TRY(cudaGetLastError());
      chunk_keys = sharded ? h->d_all_keys.as<uint8_t>() + (size_t)c0 * (size_t)keys_stride * 16 : sl.d_keys.as<uint8_t>();
      if (keys_stride > 0) {
        if (io->keys) PIPE_CUDA_TRY(cudaMemsetAsync(chunk_keys, 0, (size_t)m * (size_t)keys_stride * 16, s_k));
        PIPE_CUDA_TRY(xxh3_chain_launch(sl.d_ids.as<int32_t>(), sl.d_tok_start.as<int64_t>(), sl.d_n_tok.as<int32_t>(),
                                        chunk_keys, sl.d_key_start.as<int64_t>(), m, h->block_size, h->xxh,
                                        sl.counters + 8, s_k));
      }
      if (sharded) {
        batch_rows_kernel<<<(m + 127) / 128, 128, 0, s_k>>>(sl.d_n_blocks.as<int32_t>(), m, (int64_t)c0, keys_stride,
                                                           h->d_all_key_start.as<int64_t>(),
                                                           h->d_all_n_blocks.as<int32_t>());
        PIPE_CUDA_TRY(cudaGetLastError());
      } else if (want_match) {
        // probe + first-miss scan + routing in one kernel, between begin_read / end_read so that a publish from
        // another handle of this index waits for it (prefix_index.cuh)
        h->index->begin_read();
        const cudaError_t me = h->index->match_route(sl.d_keys.as<uint8_t>(), sl.d_key_start.as<int64_t>(),
                                                     sl.d_n_blocks.as<int32_t>(), m, h->d_inst,
                                                     sl.d_match.as<MatchOut>(), sl.d_routing.as<RoutingOut>(), s_k);
        h->index->end_read(h->index_read_ev, s_k);
        PIPE_CUDA_TRY(me);
      }
    }
    if (io->ids_u16) {
      const size_t n_ids_chunk = (size_t)m * (size_t)io->ids_stride;
      if ((rc = sl.d_ids16.reserve(n_ids_chunk * 2 + 64)) != XLLM_OK) break;
      narrow_ids_kernel<<<(unsigned)((n_ids_chunk / 8 + 256) / 256), 256, 0, s_k>>>(sl.d_ids.as<int32_t>(),
                                                                                  sl.d_ids16.as<uint16_t>(), n_ids_chunk);
      PIPE_CUDA_TRY(cudaGetLastError());
      h->last_launches += 1;
    }
    PIPE_CUDA_TRY(cudaEventRecord(sl.ev[1], s_k));
    // ---- download
    PIPE_CUDA_TRY(cudaStreamWaitEvent(s_out, sl.ev[1], 0));
    if (io->ids_u16)
      PIPE_CUDA_TRY(cudaMemcpyAsync(io->ids_u16 + (size_t)c0 * io->ids_stride, sl.d_ids16.p,
                                    (size_t)m * (size_t)io->ids_stride * 2, cudaMemcpyDeviceToHost, s_out));
    else
      PIPE_CUDA_TRY(cudaMemcpyAsync(io->ids + (size_t)c0 * io->ids_stride, sl.d_ids.p,
                                    (size_t)m * (size_t)io->ids_stride * 4, cudaMemcpyDeviceToHost, s_out));
    mark(3, s_out);
    PIPE_CUDA_TRY(cudaMemcpyAsync(io->n_ids + c0, sl.d_n_ids.p, (size_t)m * 4, cudaMemcpyDeviceToHost, s_out));
    PIPE_CUDA_TRY(cudaMemcpyAsync(io->status + c0, sl.d_status.p, (size_t)m * 4, cudaMemcpyDeviceToHost, s_out));
    if (keys_stride > 0 && io->keys)
      PIPE_CUDA_TRY(cudaMemcpyAsync(io->keys + (size_t)c0 * (size_t)keys_stride * 16, chunk_keys,
                                    (size_t)m * (size_t)keys_stride * 16, cudaMemcpyDeviceToHost, s_out));
    if (want_match && !sharded && io->match)
      PIPE_CUDA_TRY(cudaMemcpyAsync(io->match + c0, sl.d_match.p, (size_t)m * sizeof(MatchOut),
                                    cudaMemcpyDeviceToHost, s_out));
    if (want_match && !sharded && io->routing)
      PIPE_CUDA_TRY(cudaMemcpyAsync(io->routing + c0, sl.d_routing.p, (size_t)m * sizeof(RoutingOut),
                                    cudaMemcpyDeviceToHost, s_out));
    PIPE_CUDA_TRY(cudaEventRecord(sl.ev[2], s_out));
    mark(4, s_out);
    sl.busy = true;
    h->last_chunks += 1;
    h->last_launches += plan.kernels + (keys_stride > 0 || want_match ? 1 : 0) + (keys_stride > 0 ? 1 : 0) + (want_match ? 1 : 0);  // encode, prep, hash, match+route
    slot = (slot + 1) % n_slots;
    c0 = c1;
  }
#undef PIPE_CUDA_TRY
  if (sharded && rc == XLLM_OK) {
    // every chunk's hash kernel is queued on s_k ahead of this; the round synchronises s_k before it returns
    rc = h->shard->match_route(*h->index, h->index_read_ev, h->d_all_keys.as<uint8_t>(), h->d_all_key_start.as<int64_t>(),
                               h->d_all_n_blocks.as<int32_t>(), n, (int64_t)n * keys_stride, h->d_inst,
                               h->d_all_match.as<MatchOut>(), h->d_all_routing.as<RoutingOut>(), s_k);
    h->last_launches += 5;   // bucket, headers, owner probe, header gather, scan + route (+ 2 NCCL rounds)
    cudaError_t ce = cudaSuccess;
    if (rc == XLLM_OK && io->match)
      ce = cudaMemcpyAsync(io->match, h->d_all_match.p, (size_t)n * sizeof(MatchOut), cudaMemcpyDeviceToHost, s_k);
    if (rc == XLLM_OK && ce == cudaSuccess && io->routing)
      ce = cudaMemcpyAsync(io->routing, h->d_all_routing.p, (size_t)n * sizeof(RoutingOut), cudaMemcpyDeviceToHost, s_k);
    if (ce != cudaSuccess) {
      set_last_error("xllm_ingest_batch (sharded match download): %s", cudaGetErrorString(ce));
      rc = XLLM_ERR_CUDA;
    }
  }
  {
    cudaError_t e = cudaStreamSynchronize(s_out);
    cudaError_t e2 = cudaStreamSynchronize(s_k);
    cudaError_t e3 = cudaStreamSynchronize(s_in);
    if (e == cudaSuccess) e = e2;
    if (e == cudaSuccess) e = e3;
    if (e != cudaSuccess && rc == XLLM_OK) {
      set_last_error("xllm_ingest_batch: %s", cudaGetErrorString(e));
      rc = XLLM_ERR_CUDA;
    }
  }
  if (trace && rc == XLLM_OK) {
    fprintf(stderr, "# chunk m host_enqueue  h2d_begin h2d_end encode_end d2h_ids_end all_end   (ms since batch start)\n");
    for (size_t i = 0; i < rows.size(); ++i) {
      float t[5];
      for (int k = 0; k < 5; ++k) { cudaEventElapsedTime(&t[k], ev_begin, rows[i].e[k]); cudaEventDestroy(rows[i].e[k]); }
      fprintf(stderr, "%3zu %5d %8.3f  %8.3f %8.3f %8.3f %8.3f %8.3f\n", i, rows[i].m, rows[i].host_ms, t[0], t[1], t[2], t[3], t[4]);
    }
    cudaEventDestroy(ev_begin);
  }
  return rc;
}

int xllm_last_batch_stats(xllm_ingest_t h, int32_t* n_chunks, int32_t* n_kernel_launches) {
  if (!h) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  if (n_chunks) *n_chunks = h->last_chunks;
  if (n_kernel_launches) *n_kernel_launches = h->last_launches;
  return XLLM_OK;
}

int xllm_set_memo_policy(xllm_ingest_t h, int64_t persist_requests) {
  if (!h || persist_requests < 0) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  h->memo_persist_requests = persist_requests;
  return XLLM_OK;
}

int xllm_set_nfc_policy(xllm_ingest_t h, int32_t policy) {
  if (!h || (policy != XLLM_NFC_PROVE_INERT && policy != XLLM_NFC_VERIFY)) {
    xllm::set_last_error("xllm_set_nfc_policy: invalid argument");
    return XLLM_ERR_INVALID_ARG;
  }
  std::lock_guard<std::mutex> lock(h->mu);
  h->nfc_policy = policy;
  return XLLM_OK;
}

int xllm_set_pipeline(xllm_ingest_t h, int32_t chunk_requests, int64_t chunk_bytes) {
  if (!h || chunk_requests <= 0 || chunk_bytes <= 0) return XLLM_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(h->mu);
  h->pipe_chunk_req = chunk_requests;
  h->pipe_chunk_bytes = chunk_bytes;
  return XLLM_OK;
}

}  // extern "C"
