// Payload path: minibatch gather (HBM -> SMEM -> HBM through the TMA engine's
// 1-D bulk copies), ingest (push), eviction and the synthetic counter-hash fill.
//
// Replaces Replay.buffer's deepcopy + pickle.loads + np.stack
// (APE_X/ReplayMemory.py:61-116, baseline/PER.py:113) — the dominant CPU cost
// of the reference path (SURVEY.md §3.1).
#include "bulk_rows.cuh"

namespace b2rl {

// ----------------------------------------------------------------------------
// Bulk gather: the TMA row copy of bulk_rows.cuh over the minibatch, each CTA on a contiguous item range.
// CHUNK = 14 KiB (half a frame stack, 16 stages) measured best: stores of the first
// chunks overlap the loads of the later ones, and the single driving thread is not
// yet issue-bound (8 KiB chunks were 10 % slower, 28 KiB chunks 2 % slower).
// Warp 1 copies the scalar fields (action, reward, done, ...) of the CTA's share of
// the samples, so one launch assembles the whole minibatch.
// ----------------------------------------------------------------------------
constexpr int GATHER_THREADS = 64;

struct GatherParams {
  BulkRows bulk;                       // bulk (TMA) fields
  SmallField s[B2RL_MAX_FIELDS];       // small fields, copied by warp 1
  int32_t n_small;
  int64_t n;            // samples
  int64_t capacity;
  int64_t total_items;  // bulk.items_per_row * n
};

template <int CHUNK, int LAG>
__global__ void __launch_bounds__(GATHER_THREADS, 1)
k_gather_bulk(const __grid_constant__ GatherParams P, const int64_t* __restrict__ idx) {
  if (threadIdx.x >= 32) {
    // ---- warp 1: scalar fields of samples [k0, k1) ------------------------------------
    const int64_t per = (P.n + gridDim.x - 1) / gridDim.x;
    const int64_t k0 = (int64_t)blockIdx.x * per;
    const int64_t k1 = (k0 + per < P.n) ? k0 + per : P.n;
    for (int f = 0; f < P.n_small; ++f)
      copy_small_rows(P.s[f], [&](int64_t k) { return clamp_row(idx[k], P.capacity); }, k0, k1, threadIdx.x - 32,
                      32);
    return;
  }
  if (threadIdx.x != 0) return;  // a single thread drives the copy engine
  // items of this CTA: a contiguous range, so consecutive items share idx[] cache lines
  const int64_t per_cta = (P.total_items + gridDim.x - 1) / gridDim.x;
  const int64_t first = (int64_t)blockIdx.x * per_cta;
  if (first >= P.total_items) return;
  const int64_t my_items = (P.total_items - first < per_cta) ? P.total_items - first : per_cta;
  copy_rows<CHUNK, LAG>(P.bulk, [&](int64_t k) { return clamp_row(idx[k], P.capacity); }, 0, first, my_items);
}

// Generic fallback / small fields: one thread per (sample, 4-byte word or byte).
__global__ void __launch_bounds__(256)
k_gather_small(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int64_t row_bytes,
               const int64_t* __restrict__ idx, int64_t n, int64_t capacity) {
  copy_small_rows(SmallField{src, dst, row_bytes}, [&](int64_t k) { return clamp_row(idx[k], capacity); }, 0, n,
                  (int64_t)blockIdx.x * blockDim.x + threadIdx.x, (int64_t)gridDim.x * blockDim.x);
}

// LDG.128/STG.128 reference implementation of the big-row gather (kept for the
// A/B comparison with the bulk-copy gather, selectable with B2RL_GATHER=ldg).
__global__ void __launch_bounds__(256)
k_gather_ldg(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int64_t row_bytes,
             const int64_t* __restrict__ idx, int64_t n, int64_t capacity) {
  const int64_t k = blockIdx.x;
  if (k >= n) return;
  const int64_t row = clamp_row(idx[k], capacity);
  const int4* s = reinterpret_cast<const int4*>(src + row * row_bytes);
  int4* d = reinterpret_cast<int4*>(dst + k * row_bytes);
  const int64_t nv = row_bytes >> 4;
  for (int64_t i = threadIdx.x; i < nv; i += 4 * 256) {
    int4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (i + u * 256 < nv) v[u] = __ldg(s + i + u * 256);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (i + u * 256 < nv) d[i + u * 256] = v[u];
  }
}

// ----------------------------------------------------------------------------
// Synthetic fill: word w of slot s of field f =
//   lowbias32(seed ^ f*0x9E3779B9 ^ (uint32)s*2654435761 ^ (uint32)w*2246822519)
// (tail bytes of a row whose size is not a multiple of 4 take the low bytes).
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_fill_hash(uint8_t* __restrict__ base, int64_t row_bytes, int64_t n_rows, uint32_t seed, uint32_t fsalt) {
  const int64_t words_per_row = (row_bytes + 3) >> 2;
  const int64_t total = n_rows * words_per_row;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = t / words_per_row, w = t - s * words_per_row;
    const uint32_t v = lowbias32(seed ^ fsalt ^ ((uint32_t)s * 2654435761U) ^ ((uint32_t)w * 2246822519U));
    uint8_t* p = base + s * row_bytes + w * 4;
    const int64_t left = row_bytes - w * 4;
    if (left >= 4 && ((row_bytes & 3) == 0)) {
      *reinterpret_cast<uint32_t*>(p) = v;
    } else {
      for (int b = 0; b < 4 && b < left; ++b) p[b] = (uint8_t)(v >> (8 * b));
    }
  }
}

}  // namespace b2rl

using namespace b2rl;

int b2rl_tree_update_impl(b2rl_replay* h, const int64_t* idx_dev, int64_t ring_start,
                          const float* vals_dev, float const_val, int64_t n, cudaStream_t st,
                          bool publish_size_too);

static int gather_chunk() {
  static int chunk = -1;
  if (chunk < 0) {
    const char* e = getenv("B2RL_GATHER_CHUNK");   // 28672 (8 stages) | 14336 (16) | 7168 (32 -> 28 used)
    chunk = e ? atoi(e) : 14336;
    if (chunk != 28672 && chunk != 14336 && chunk != 8192) chunk = 14336;
  }
  return chunk;
}

static int gather_mode() {
  static int mode = -1;
  if (mode < 0) {
    const char* e = getenv("B2RL_GATHER");
    mode = (e && e[0] == 'l') ? 1 : 0;  // "ldg" -> 1, default bulk/TMA -> 0
  }
  return mode;
}

// b2rl_replay_gather, and for a dedup replay b2rl_replay_gather_planes: stacks_out (2 entries, or nullptr) receives
// the frame stacks of planes 0-3 / 4-7 (Ape-X), or in its first entry the R-frame strips of a strip handle, copied
// as plane rows by the same launch.
static int gather_run(b2rl_replay* h, const int64_t* idx_dev, int64_t n, void* const* stacks_out,
                      void* const* out_fields_dev, cudaStream_t st) {
  GatherParams P{};
  P.n = n;
  P.capacity = h->capacity;
  if (stacks_out != nullptr) {
    const int32_t* planes = (const int32_t*)h->field[dedup_planes_field(h)];
    const int R = dedup_strip_frames(h);
    if (R > 0) {
      B2RL_REQUIRE(stacks_out[1] == nullptr, "a strip handle has one frame output: stacks_out_dev[1] must be NULL");
      B2RL_REQUIRE((uintptr_t)stacks_out[0] % 16 == 0, "frame strip outputs must be 16-byte aligned");
      if (stacks_out[0] != nullptr && dedup_pool_on_host(h)) {   // never the TMA row copy: hostrows.cu's gather
        const int rc = gather_host_planes(h, idx_dev, n, (uint8_t*)stacks_out[0], st);
        if (rc != B2RL_OK) return rc;
      } else if (stacks_out[0] != nullptr && dedup_pool_coded(h)) {   // decoded from the unit ring (dedup.cu)
        const int rc = gather_coded_planes(h, idx_dev, n, (uint8_t*)stacks_out[0], nullptr, st);
        if (rc != B2RL_OK) return rc;
      } else if (stacks_out[0] != nullptr) {
        P.bulk.add_planes(dedup_pool(h), planes, R, 0, R, (uint8_t*)stacks_out[0]);
      }
    } else if (dedup_pool_coded(h)) {   // s and s' decoded from the unit ring (dedup.cu)
      const int rc = gather_coded_planes(h, idx_dev, n, (uint8_t*)stacks_out[0], (uint8_t*)stacks_out[1], st);
      if (rc != B2RL_OK) return rc;
    } else {
      for (int i = 0; i < 2; ++i) {
        B2RL_REQUIRE((uintptr_t)stacks_out[i] % 16 == 0, "frame stack outputs must be 16-byte aligned");
        if (stacks_out[i] != nullptr) P.bulk.add_planes(dedup_pool(h), planes, 8, 4 * i, 4, (uint8_t*)stacks_out[i]);
      }
    }
  }
  for (int f = 0; f < h->n_fields; ++f) {
    uint8_t* out = out_fields_dev ? (uint8_t*)out_fields_dev[f] : nullptr;
    if (out == nullptr || (stacks_out != nullptr && f == dedup_planes_field(h))) continue;
    if (h->on_host[f]) {                  // never the TMA row copy: the 16-byte load gather of hostrows.cu
      const int rc = gather_host_rows(h, f, idx_dev, n, out, st);
      if (rc != B2RL_OK) return rc;
      continue;
    }
    const int64_t rb = h->field_bytes[f];
    const bool big = rb >= 1024;
    const bool bulk = is_bulk_row(rb) && ((uintptr_t)out % 16 == 0) && ((uintptr_t)h->field[f] % 16 == 0);
    if (bulk && gather_mode() == 0) {
      P.bulk.add(h->field[f], out, rb, gather_chunk());
    } else if (bulk) {
      k_gather_ldg<<<(unsigned)n, 256, 0, st>>>(h->field[f], out, rb, idx_dev, n, h->capacity);
      count_launch();
    } else if (!big && ((rb % 4 != 0) || (((uintptr_t)out % 4 == 0) && ((uintptr_t)h->field[f] % 4 == 0)))) {
      P.s[P.n_small++] = SmallField{h->field[f], out, rb};
    } else {
      const int64_t units = (rb % 4 == 0 && (uintptr_t)out % 4 == 0) ? n * (rb / 4) : n * rb;
      k_gather_small<<<(unsigned)((units + 255) / 256), 256, 0, st>>>(h->field[f], out, rb, idx_dev, n,
                                                                     h->capacity);
      count_launch();
    }
  }
  if (P.bulk.n > 0 || P.n_small > 0) {
    P.total_items = P.bulk.items_per_row * n;
    const int dev = h->device;
    int sms = 0;
    B2RL_CUDA(sm_count(dev, &sms));
    B2RL_CUDA((set_max_dynamic_smem<k_gather_bulk<28672, 1>>(dev, BULK_RING_BYTES)));
    B2RL_CUDA((set_max_dynamic_smem<k_gather_bulk<14336, 3>>(dev, BULK_RING_BYTES)));
    B2RL_CUDA((set_max_dynamic_smem<k_gather_bulk<8192, 6>>(dev, BULK_RING_BYTES)));
    int64_t grid = sms;
    const int64_t work = P.total_items > n ? P.total_items : n;
    if (grid > work) grid = work;
    switch (gather_chunk()) {
      case 28672: k_gather_bulk<28672, 1><<<(unsigned)grid, GATHER_THREADS, BULK_RING_BYTES, st>>>(P, idx_dev); break;
      case 8192:  k_gather_bulk<8192, 6><<<(unsigned)grid, GATHER_THREADS, BULK_RING_BYTES, st>>>(P, idx_dev); break;
      default:    k_gather_bulk<14336, 3><<<(unsigned)grid, GATHER_THREADS, BULK_RING_BYTES, st>>>(P, idx_dev); break;
    }
    count_launch();
  }
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_replay_gather(b2rl_replay* h, const int64_t* idx_dev, int64_t n,
                                  void* const* out_fields_dev, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0, "negative n");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(idx_dev != nullptr && out_fields_dev != nullptr, "null argument");
  DeviceGuard g(h->device);
  return gather_run(h, idx_dev, n, nullptr, out_fields_dev, (cudaStream_t)stream);
}

extern "C" int b2rl_replay_gather_planes(b2rl_replay* h, const int64_t* idx_dev, int64_t n, void* const* stacks_out_dev,
                                         void* const* out_fields_dev, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(h->dedup != nullptr, "not a frame-deduplicated replay (b2rl_dedup_attach)");
  B2RL_REQUIRE(n >= 0, "negative n");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(idx_dev != nullptr && stacks_out_dev != nullptr, "null argument");
  DeviceGuard g(h->device);
  return gather_run(h, idx_dev, n, stacks_out_dev, out_fields_dev, (cudaStream_t)stream);
}

extern "C" int b2rl_replay_fill_hash(b2rl_replay* h, int64_t n, uint32_t seed, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0 && n <= h->capacity, "n out of range");
  B2RL_REQUIRE(h->dedup == nullptr, "a frame-deduplicated replay holds pool ids, not hashable payload");
  DeviceGuard g(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  for (int f = 0; f < h->n_fields; ++f) {
    const int64_t words = n * ((h->field_bytes[f] + 3) / 4);
    if (words == 0) continue;
    int64_t blocks = (words + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;   // 32 CTAs per SM of an H100
    k_fill_hash<<<(unsigned)blocks, 256, 0, st>>>(h->field[f], h->field_bytes[f], n, seed,
                                                  (uint32_t)f * 0x9E3779B9U);
    count_launch();
  }
  B2RL_CHECK_LAUNCH();
  h->size = n;
  h->head = (n == h->capacity) ? 0 : n;
  return publish_size(h, st);
}

int b2rl::copy_ring_range(b2rl_replay* h, const void* const* fields_src, int64_t start, int64_t n, cudaStream_t st) {
  const int64_t first = (start + n <= h->capacity) ? n : (h->capacity - start);  // before the wrap
  for (int f = 0; f < h->n_fields; ++f) {
    const uint8_t* src = (const uint8_t*)fields_src[f];
    if (src == nullptr) continue;
    const int64_t rb = h->field_bytes[f];
    if (h->on_host[f]) {
      int rc = copy_into_host_field(h, f, start, src, first * rb, st);
      if (rc == B2RL_OK && first < n) rc = copy_into_host_field(h, f, 0, src + first * rb, (n - first) * rb, st);
      if (rc != B2RL_OK) return rc;
      continue;
    }
    B2RL_CUDA(cudaMemcpyAsync(h->field[f] + start * rb, src, (size_t)(first * rb), cudaMemcpyDefault, st));
    if (first < n)
      B2RL_CUDA(cudaMemcpyAsync(h->field[f], src + first * rb, (size_t)((n - first) * rb), cudaMemcpyDefault, st));
  }
  return B2RL_OK;
}

int b2rl::publish(b2rl_replay* h, const float* prios_dev, int64_t n, cudaStream_t st) {
  h->size = (h->size + n > h->capacity) ? h->capacity : h->size + n;   // published by the update kernel itself
  int rc = b2rl_tree_update_impl(h, nullptr, h->head, prios_dev, 0.0f, n, st, true);
  if (rc != B2RL_OK) return rc;
  h->head = (h->head + n) % h->capacity;
  return B2RL_OK;
}

// The n slots at head are about to be overwritten: their records can no longer be sampled.
static int retire(b2rl_replay* h, int64_t n, cudaStream_t st) {
  const int64_t overwritten = h->size + n - h->capacity;
  if (overwritten > 0) h->size -= overwritten;
  return b2rl_tree_update_impl(h, nullptr, h->head, nullptr, 0.0f, n, st, overwritten > 0);
}

extern "C" int b2rl_replay_push(b2rl_replay* h, const void* const* fields_src, const float* prios,
                                int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0 && n <= h->capacity, "n out of range (0..capacity)");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(prios != nullptr, "null priorities");
  B2RL_REQUIRE(h->n_fields == 0 || fields_src != nullptr, "null fields");
  B2RL_REQUIRE(h->dedup == nullptr, "a frame-deduplicated replay takes its records through b2rl_dedup_push");
  DeviceGuard g(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = check_host_sources(h, fields_src);
  if (rc != B2RL_OK) return rc;
  rc = copy_ring_range(h, fields_src, h->head, n, st);
  if (rc != B2RL_OK) return rc;
  B2RL_CUDA(cudaMemcpyAsync(h->scratch_val, prios, (size_t)n * sizeof(float), cudaMemcpyDefault, st));
  return publish(h, h->scratch_val, n, st);
}

extern "C" int b2rl_replay_reserve(b2rl_replay* h, int64_t n, int64_t* start_slot, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 1 && n <= h->capacity, "n out of range (1..capacity)");
  B2RL_REQUIRE(h->reserved == 0, "a reservation is already pending (call b2rl_replay_commit first)");
  B2RL_REQUIRE(h->dedup == nullptr, "a frame-deduplicated replay takes its records through b2rl_dedup_push");
  DeviceGuard g(h->device);
  int rc = retire(h, n, (cudaStream_t)stream);
  if (rc != B2RL_OK) return rc;
  h->reserved = n;
  if (start_slot) *start_slot = h->head;
  return B2RL_OK;
}

extern "C" int b2rl_replay_copy_payload(b2rl_replay* h, const void* const* fields_src, int64_t start_slot,
                                        int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr && fields_src != nullptr, "null argument");
  B2RL_REQUIRE(n >= 1 && n <= h->capacity && start_slot >= 0 && start_slot < h->capacity, "range out of bounds");
  DeviceGuard g(h->device);
  const int rc = check_host_sources(h, fields_src);
  if (rc != B2RL_OK) return rc;
  return copy_ring_range(h, fields_src, start_slot, n, (cudaStream_t)stream);
}

extern "C" int b2rl_replay_commit(b2rl_replay* h, const float* prios, int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr && prios != nullptr, "null argument");
  B2RL_REQUIRE(n >= 1 && n == h->reserved, "commit size must equal the pending reservation");
  DeviceGuard g(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  B2RL_CUDA(cudaMemcpyAsync(h->scratch_val, prios, (size_t)n * sizeof(float), cudaMemcpyDefault, st));
  int rc = publish(h, h->scratch_val, n, st);
  if (rc != B2RL_OK) return rc;
  h->reserved = 0;
  return B2RL_OK;
}

// One call per learner iteration for a steady ingest: publish the batch whose host->device copy was started by
// the PREVIOUS call (the learner stream waits for that copy's event, then writes its priorities: the records
// become sampleable), then retire the slots of the NEXT batch and start its copy on the library's own copy
// stream — which therefore overlaps whatever the caller enqueues on `stream` next (the learner step).
// The priorities travel with the payload and wait in device memory, so no host buffer has to outlive its copy
// beyond the next call.  fields_src == NULL flushes: publishes the pending batch and starts nothing.
extern "C" int b2rl_replay_ingest_pipelined(b2rl_replay* h, const void* const* fields_src, const float* prios_src,
                                            int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(fields_src == nullptr || (n >= 1 && n <= h->capacity && prios_src != nullptr), "bad batch");
  B2RL_REQUIRE(h->dedup == nullptr, "a frame-deduplicated replay takes its records through b2rl_dedup_push");
  DeviceGuard g(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  {
    const int rc = check_host_sources(h, fields_src);
    if (rc != B2RL_OK) return rc;
  }
  if (h->ingest_stream == nullptr) {
    B2RL_CUDA(cudaStreamCreateWithFlags(&h->ingest_stream, cudaStreamNonBlocking));
    B2RL_CUDA(cudaEventCreateWithFlags(&h->ev_reserved, cudaEventDisableTiming));
    B2RL_CUDA(cudaEventCreateWithFlags(&h->ev_copied, cudaEventDisableTiming));
  }
  if (h->pipe_n > 0) {                      // 1. publish the batch in flight
    B2RL_REQUIRE(h->reserved == h->pipe_n, "pipelined ingest mixed with reserve/commit");
    B2RL_CUDA(cudaStreamWaitEvent(st, h->ev_copied, 0));
    int rc = publish(h, h->pipe_prios, h->pipe_n, st);
    if (rc != B2RL_OK) return rc;
    h->reserved = 0;
    h->pipe_n = 0;
    // the copy stream must not overwrite pipe_prios before this update has read it
    B2RL_CUDA(cudaEventRecord(h->ev_reserved, st));
    B2RL_CUDA(cudaStreamWaitEvent(h->ingest_stream, h->ev_reserved, 0));
  }
  if (fields_src == nullptr) return B2RL_OK;
  B2RL_REQUIRE(h->reserved == 0, "a reservation is already pending (call b2rl_replay_commit first)");
  if (h->pipe_cap < n) {                    // (re)grow the priority staging; rare, synchronous
    B2RL_CUDA(cudaStreamSynchronize(h->ingest_stream));
    B2RL_CUDA(cudaStreamSynchronize(st));
    if (h->pipe_prios) cudaFree(h->pipe_prios);
    h->pipe_prios = nullptr;
    B2RL_CUDA(cudaMalloc((void**)&h->pipe_prios, sizeof(float) * (size_t)n));
    h->pipe_cap = n;
  }
  int rc = retire(h, n, st);                // 2. retire the slots about to be overwritten
  if (rc != B2RL_OK) return rc;
  h->reserved = n;
  h->pipe_n = n;
  // 3. payload + priorities on the copy stream, behind the retirement
  B2RL_CUDA(cudaEventRecord(h->ev_reserved, st));
  B2RL_CUDA(cudaStreamWaitEvent(h->ingest_stream, h->ev_reserved, 0));
  rc = copy_ring_range(h, fields_src, h->head, n, h->ingest_stream);
  if (rc != B2RL_OK) return rc;
  B2RL_CUDA(cudaMemcpyAsync(h->pipe_prios, prios_src, (size_t)n * sizeof(float), cudaMemcpyDefault, h->ingest_stream));
  B2RL_CUDA(cudaEventRecord(h->ev_copied, h->ingest_stream));
  return B2RL_OK;
}

extern "C" int b2rl_replay_evict(b2rl_replay* h, int64_t delta, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(delta >= 0 && delta <= h->size, "delta out of range (0..size)");
  if (delta == 0) return B2RL_OK;
  DeviceGuard g(h->device);
  // oldest record lives at (head - size) mod capacity
  int64_t tail = h->head - h->size;
  if (tail < 0) tail += h->capacity;
  h->size -= delta;
  return b2rl_tree_update_impl(h, nullptr, tail, nullptr, 0.0f, delta, (cudaStream_t)stream, true);
}
