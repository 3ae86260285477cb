// Device serve ring of the stand-alone replay server (include/b2rl.h, "Device serve ring"): layout arithmetic,
// allocation / CUDA IPC export and import, and k_serve_fill — draw + IS weights + scalar fetch + small-row copy +
// TMA bulk copy of the frame rows of one minibatch into a ring slot in ONE launch.
//
// Replaces ReplayServer.buffer's sample -> gather -> .cpu() -> pickle -> RPUSH and Replay_Server.sample's
// pickle.loads -> host-to-device copy (APE_X/ReplayServer.py:65-114, APE_X/ReplayMemory.py:251-257).
#include "bulk_rows.cuh"
#include "tree.cuh"
#include "uniform.cuh"

#include <new>

namespace b2rl {

constexpr int SERVE_THREADS = 128;   // draws per CTA at most; warp 0's lane 0 then drives the copy engine

// Fields of a served record whose rows are neither bulk rows nor 1/2/4/8-byte scalars (SmallRows) are copied by
// warps 1..3 of the CTA while thread 0 drives the TMA row copy.

// BY_ITEMS (fewer draws than SMs): CTA c owns a contiguous range of the minibatch's copy items (draw-major, then
// field, then chunk: the items of copy_rows), as k_gather_bulk's CTAs do, so the copy still spreads over
// every SM.  Its threads draw every draw the range touches; a draw is a pure function of the Philox counter (and the
// tree), so each CTA that draws k gets the same slot.  The CTA that holds draw k's first item owns it and alone
// writes idx[k], w[k] and its scalar and small rows.  Otherwise CTA c owns draws [c*per, (c+1)*per) whole: for Ape-X
// B = 512 the two splits give the same partition, and the item split's extra index arithmetic measured 1.7 % slower.  Thread 0 copies the range's bulk items with the TMA row copy of bulk_rows.cuh
// (k_gather_bulk's default geometry: 14 KiB chunks, 16 stages, lag 3), warps 1..3 copy the owned draws' small rows,
// then the last CTA to finish writes the header.  A record without bulk fields counts one item per draw.
// draw(seed, offset, k, owned, row) stores the replay row of draw k in `row`; an owned draw also writes its idx / w /
// scalars.
// TIME_MAJOR: step t of draw k goes to output row t * n + k (bulk rows and the small rows of T 4-byte steps).
template <bool BY_ITEMS, bool TIME_MAJOR, int CHUNK, class Draw>
__device__ __forceinline__ void serve_fill(const BulkRows& P, const SmallRows& rows, uint64_t* __restrict__ rng_state,
                                           int64_t n, const Draw& draw, uint64_t* __restrict__ header, uint64_t seq,
                                           unsigned int* __restrict__ done_ticket) {
  __shared__ int64_t s_row[SERVE_THREADS];
  const int tid = threadIdx.x;
  uint64_t seed, offset;
  rng_stream_take(rng_state, n, seed, offset);      // every block, exactly as k_tree_sample
  const int64_t ipr = P.n > 0 ? P.items_per_row : 1;
  // items [first, first + items); draws touched [k_lo, k_hi), owned [k_own, k_hi); k_hi - k_lo <= SERVE_THREADS
  int64_t first, items, k_lo, k_own, k_hi;
  if (BY_ITEMS) {
    const int64_t total = n * ipr;
    const int64_t per = (total + gridDim.x - 1) / gridDim.x;
    first = (int64_t)blockIdx.x * per;
    items = (first >= total) ? 0 : ((total - first < per) ? total - first : per);
    k_lo = first / ipr;
    k_own = (first + ipr - 1) / ipr;
    k_hi = (items > 0) ? (first + items + ipr - 1) / ipr : k_lo;
  } else {
    const int64_t per = (n + gridDim.x - 1) / gridDim.x;
    k_lo = k_own = (int64_t)blockIdx.x * per;
    k_hi = (k_lo >= n) ? k_lo : ((n - k_lo < per) ? n : k_lo + per);
    first = k_lo * ipr;
    items = (k_hi - k_lo) * ipr;
  }
  if (tid < k_hi - k_lo) {
    const int64_t k = k_lo + tid;
    draw(seed, offset, k, k >= k_own, s_row[tid]);
  }
  __syncthreads();
  if (items > 0) {
    if (tid == 0 && P.n > 0) {
      copy_rows<CHUNK, 3, TIME_MAJOR>(P, [](int64_t i) { return s_row[i]; }, k_lo, first - k_lo * ipr, items, n);
    } else if (tid >= 32) {
      for (int f = 0; f < rows.n; ++f) {
        if (TIME_MAJOR)
          copy_small_rows_time_major(rows.f[f], [&](int64_t k) { return s_row[k - k_lo]; }, k_own, k_hi, n,
                                     tid - 32, SERVE_THREADS - 32);
        else
          copy_small_rows(rows.f[f], [&](int64_t k) { return s_row[k - k_lo]; }, k_own, k_hi, tid - 32,
                          SERVE_THREADS - 32);
      }
    }
  }
  // header last: written by the last CTA to get here, after every CTA's copies have completed
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(done_ticket, 1u) == gridDim.x - 1) {
      __threadfence();
      header[0] = seq;
      header[1] = (uint64_t)n;
      *done_ticket = 0u;       // re-armed for the next fill
    }
  }
}

// The prioritized fill (Ape-X, R2D2): sum-tree descent + IS weights, batch-major slot.
template <bool BY_ITEMS>
__global__ void __launch_bounds__(SERVE_THREADS, 1)
k_serve_fill(const __grid_constant__ TreeView t, const __grid_constant__ BulkRows P, SmallFields small,
             const __grid_constant__ SmallRows rows, uint64_t* __restrict__ rng_state, int64_t n, int64_t capacity,
             const float* __restrict__ n_valid_dev, float beta, const float* __restrict__ max_w_ext,
             int64_t* __restrict__ idx_out, float* __restrict__ w_out, uint64_t* __restrict__ header, uint64_t seq,
             unsigned int* __restrict__ done_ticket) {
  serve_fill<BY_ITEMS, false, 14336>(P, rows, rng_state, n,
                                     [&](uint64_t seed, uint64_t offset, int64_t k, bool own, int64_t& row) {
    double root, picked;
    const int64_t j = tree_draw(t, philox_u01(seed, offset + (uint64_t)k), root, picked);
    row = clamp_row(j, capacity);   // the row b2rl_replay_gather would copy
    if (own) {
      idx_out[k] = j;
      fetch_small(small, j, k);
      const float s32 = (float)root;
      w_out[k] = is_weight(t, s32, __fdiv_rn((float)picked, s32), n_valid_dev, beta, max_w_ext);
    }
  }, header, seq, done_ticket);
}

// The IMPALA fill: the uniform draw without replacement of uniform.cuh, time-major slot.
constexpr int UNIFORM_CHUNK = 14112;   // half an 84x84x4 frame stack: no chunk of a time-major frame row straddles two steps

template <bool BY_ITEMS>
__global__ void __launch_bounds__(SERVE_THREADS, 1)
k_serve_fill_uniform(const __grid_constant__ BulkRows P, SmallFields small, const __grid_constant__ SmallRows rows,
                     uint64_t* __restrict__ rng_state, int64_t n, UniformDraw u, int64_t* __restrict__ idx_out,
                     uint64_t* __restrict__ header, uint64_t seq, unsigned int* __restrict__ done_ticket) {
  serve_fill<BY_ITEMS, true, UNIFORM_CHUNK>(P, rows, rng_state, n,
                                            [&](uint64_t seed, uint64_t offset, int64_t k, bool own, int64_t& row) {
    uint32_t key[4];
    philox4x32_10(offset, seed, key);
    const int64_t j = uniform_row(u, key, k);
    row = j;
    if (own) {
      idx_out[k] = j;
      fetch_small(small, j, k);
    }
  }, header, seq, done_ticket);
}

__global__ void __launch_bounds__(256)
k_serve_put_update(uint64_t* __restrict__ header, int64_t* __restrict__ idx_dst, float* __restrict__ prio_dst,
                   const int64_t* __restrict__ idx_src, const float* __restrict__ prio_src, int64_t n, uint64_t seq) {
  for (int64_t k = threadIdx.x; k < n; k += blockDim.x) {
    idx_dst[k] = idx_src[k];
    prio_dst[k] = prio_src[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    header[0] = seq;
    header[1] = (uint64_t)n;
  }
}

// k_serve_bind: hand a filled minibatch slot to a captured learner step.  The step's graph reads fixed buffers and a
// frame table; the bind copies the slot's small arrays into those buffers (CTA j copies job j) and writes the device
// addresses of the frame fields' rows into the table entries (CTA 0), so conv_1 reads the frames in the slot itself.
struct BindCopy {
  const uint8_t* src;
  uint8_t* dst;
  int64_t bytes;
};
struct BindJobs {
  BindCopy copy[3 + B2RL_MAX_FIELDS];         // header, idx, w, then the copied fields
  const uint8_t* addr[B2RL_MAX_FIELDS];       // rows of a frame field ...
  const uint8_t** entry[B2RL_MAX_FIELDS];     // ... and the table entry that receives their address
  int32_t n_entries;
};

__global__ void __launch_bounds__(256)
k_serve_bind(const __grid_constant__ BindJobs J) {
  if (blockIdx.x == 0 && threadIdx.x < J.n_entries) *J.entry[threadIdx.x] = J.addr[threadIdx.x];
  const BindCopy c = J.copy[blockIdx.x];
  if ((((uintptr_t)c.src | (uintptr_t)c.dst | (uintptr_t)c.bytes) & 15) == 0) {
    const uint4* s = reinterpret_cast<const uint4*>(c.src);
    uint4* d = reinterpret_cast<uint4*>(c.dst);
    for (int64_t i = threadIdx.x; i < c.bytes / 16; i += blockDim.x) d[i] = s[i];
  } else {
    for (int64_t i = threadIdx.x; i < c.bytes; i += blockDim.x) c.dst[i] = c.src[i];
  }
}

}  // namespace b2rl

using namespace b2rl;

struct b2rl_serve_ring {
  int device = 0;
  bool owned = false;                  // created here (destroy) or mapped through IPC (close)
  b2rl_serve_layout L = {};
  uint8_t* base = nullptr;
  unsigned int* done_ticket = nullptr; // k_serve_fill's last-CTA counter (owner only)
};

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

extern "C" int b2rl_serve_layout_init(int64_t batch, int32_t slots, int32_t n_fields, const int64_t* field_bytes,
                                      b2rl_serve_layout* out) {
  B2RL_REQUIRE(out != nullptr, "null out");
  B2RL_REQUIRE(batch >= 1 && batch <= (1LL << 24), "batch out of range (1..2^24)");
  B2RL_REQUIRE(slots >= 1 && slots <= 1024, "slots out of range (1..1024)");
  B2RL_REQUIRE(n_fields >= 0 && n_fields <= B2RL_MAX_FIELDS, "n_fields out of range");
  B2RL_REQUIRE(n_fields == 0 || field_bytes != nullptr, "null field_bytes");
  b2rl_serve_layout L;
  memset(&L, 0, sizeof(L));
  L.batch = batch;
  L.slots = slots;
  L.n_fields = n_fields;
  int64_t off = 16;                                  // header {seq, n}
  L.idx_off = off;  off = align_up(off + 8 * batch, 16);
  L.w_off = off;    off = align_up(off + 4 * batch, 16);
  for (int f = 0; f < n_fields; ++f) {
    B2RL_REQUIRE(field_bytes[f] >= 1, "field_bytes must be >= 1");
    L.field_bytes[f] = field_bytes[f];
    L.field_off[f] = off;
    off = align_up(off + field_bytes[f] * batch, 16);
  }
  L.slot_bytes = align_up(off, 128);
  off = 16;
  L.upd_idx_off = off;  off = align_up(off + 8 * batch, 16);
  L.upd_prio_off = off; off = align_up(off + 4 * batch, 16);
  L.upd_slot_bytes = align_up(off, 128);
  L.upd_base = (int64_t)slots * L.slot_bytes;
  L.total_bytes = L.upd_base + (int64_t)slots * L.upd_slot_bytes;
  *out = L;
  return B2RL_OK;
}

// The fields a ring slot carries for replay h: its own fields, except that a frame-deduplicated replay's planes field
// becomes two frame stacks (planes 0-3, then 4-7), so the slot holds the stack store's record layout; a strip
// handle's becomes the R-frame strip field, so the slot holds the strip store's.  -> count.
static int served_fields(const b2rl_replay* h, int64_t* bytes) {
  int n = 0;
  for (int f = 0; f < h->n_fields; ++f) {
    if (h->dedup != nullptr && f == dedup_planes_field(h) && dedup_strip_frames(h) > 0) {
      bytes[n++] = (int64_t)dedup_strip_frames(h) * PLANE_BYTES;
    } else if (h->dedup != nullptr && f == dedup_planes_field(h)) {
      bytes[n++] = 4 * PLANE_BYTES;
      bytes[n++] = 4 * PLANE_BYTES;
    } else {
      bytes[n++] = h->field_bytes[f];
    }
  }
  return n;
}

extern "C" int b2rl_serve_ring_create(b2rl_replay* h, int64_t batch, int32_t slots, b2rl_serve_ring** out) {
  B2RL_REQUIRE(h != nullptr && out != nullptr, "null argument");
  B2RL_REQUIRE(h->dedup == nullptr || h->n_fields < B2RL_MAX_FIELDS, "too many fields to serve");
  b2rl_serve_layout L;
  int64_t bytes[B2RL_MAX_FIELDS];
  int rc = b2rl_serve_layout_init(batch, slots, served_fields(h, bytes), bytes, &L);
  if (rc != B2RL_OK) return rc;
  DeviceGuard g(h->device);
  b2rl_serve_ring* r = new (std::nothrow) b2rl_serve_ring();
  if (!r) { set_error("out of host memory"); return B2RL_ERR_NOMEM; }
  r->device = h->device;
  r->owned = true;
  r->L = L;
  cudaError_t e = cudaMalloc((void**)&r->base, (size_t)L.total_bytes);
  if (e == cudaSuccess) e = cudaMalloc((void**)&r->done_ticket, sizeof(unsigned int));
  if (e == cudaSuccess) e = cudaMemset(r->base, 0, (size_t)L.total_bytes);
  if (e == cudaSuccess) e = cudaMemset(r->done_ticket, 0, sizeof(unsigned int));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error("serve ring of %lld bytes: %s", (long long)L.total_bytes, cudaGetErrorString(e));
    if (r->base) cudaFree(r->base);
    if (r->done_ticket) cudaFree(r->done_ticket);
    delete r;
    cudaGetLastError();
    return B2RL_ERR_NOMEM;
  }
  *out = r;
  return B2RL_OK;
}

extern "C" int b2rl_serve_ring_layout(const b2rl_serve_ring* r, b2rl_serve_layout* out) {
  B2RL_REQUIRE(r != nullptr && out != nullptr, "null argument");
  *out = r->L;
  return B2RL_OK;
}

extern "C" int b2rl_serve_ring_export(const b2rl_serve_ring* r, void* handle_out) {
  B2RL_REQUIRE(r != nullptr && handle_out != nullptr, "null argument");
  B2RL_REQUIRE(r->owned, "only the ring's owner can export it");
  static_assert(sizeof(cudaIpcMemHandle_t) == B2RL_IPC_HANDLE_BYTES, "IPC handle size");
  DeviceGuard g(r->device);
  cudaIpcMemHandle_t hd;
  B2RL_CUDA(cudaIpcGetMemHandle(&hd, r->base));
  memcpy(handle_out, &hd, sizeof(hd));
  return B2RL_OK;
}

extern "C" int b2rl_serve_ring_open(const void* handle, const b2rl_serve_layout* layout, int32_t device,
                                    b2rl_serve_ring** out) {
  B2RL_REQUIRE(handle != nullptr && layout != nullptr && out != nullptr, "null argument");
  B2RL_REQUIRE(layout->n_fields >= 0 && layout->n_fields <= B2RL_MAX_FIELDS, "n_fields out of range");
  b2rl_serve_layout L;
  int rc = b2rl_serve_layout_init(layout->batch, (int32_t)layout->slots, (int32_t)layout->n_fields,
                                  layout->field_bytes, &L);
  if (rc != B2RL_OK) return rc;
  B2RL_REQUIRE(memcmp(&L, layout, sizeof(L)) == 0, "layout does not match the ring arithmetic of this library");
  int ndev = 0;
  B2RL_CUDA(cudaGetDeviceCount(&ndev));
  B2RL_REQUIRE(device >= 0 && device < ndev, "no such CUDA device");
  DeviceGuard g(device);
  cudaIpcMemHandle_t hd;
  memcpy(&hd, handle, sizeof(hd));
  void* p = nullptr;
  B2RL_CUDA(cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
  b2rl_serve_ring* r = new (std::nothrow) b2rl_serve_ring();
  if (!r) { cudaIpcCloseMemHandle(p); set_error("out of host memory"); return B2RL_ERR_NOMEM; }
  r->device = device;
  r->owned = false;
  r->L = L;
  r->base = (uint8_t*)p;
  *out = r;
  return B2RL_OK;
}

extern "C" int b2rl_serve_ring_close(b2rl_serve_ring* r) {
  if (!r) return B2RL_OK;
  B2RL_REQUIRE(!r->owned, "a created ring is released with b2rl_serve_ring_destroy");
  DeviceGuard g(r->device);
  const cudaError_t e = cudaIpcCloseMemHandle(r->base);
  delete r;
  B2RL_CUDA(e);
  return B2RL_OK;
}

extern "C" int b2rl_serve_ring_destroy(b2rl_serve_ring* r) {
  if (!r) return B2RL_OK;
  B2RL_REQUIRE(r->owned, "an opened ring is released with b2rl_serve_ring_close");
  DeviceGuard g(r->device);
  cudaDeviceSynchronize();
  cudaFree(r->base);
  cudaFree(r->done_ticket);
  delete r;
  return B2RL_OK;
}

extern "C" int b2rl_serve_slot_ptrs(const b2rl_serve_ring* r, int32_t slot, void** batch_out, void** update_out) {
  B2RL_REQUIRE(r != nullptr, "null ring");
  B2RL_REQUIRE(slot >= 0 && slot < r->L.slots, "slot out of range");
  const b2rl_serve_layout& L = r->L;
  if (batch_out) {
    uint8_t* s = r->base + (int64_t)slot * L.slot_bytes;
    batch_out[0] = s;
    batch_out[1] = s + L.idx_off;
    batch_out[2] = s + L.w_off;
    for (int f = 0; f < L.n_fields; ++f) batch_out[3 + f] = s + L.field_off[f];
  }
  if (update_out) {
    uint8_t* u = r->base + L.upd_base + (int64_t)slot * L.upd_slot_bytes;
    update_out[0] = u;
    update_out[1] = u + L.upd_idx_off;
    update_out[2] = u + L.upd_prio_off;
  }
  return B2RL_OK;
}

// What both fills check before anything is launched: the ring was created for this replay, on its device.
static int fill_slot_ptrs(b2rl_replay* h, b2rl_serve_ring* r, int32_t slot, void** ptrs) {
  B2RL_REQUIRE(h != nullptr && r != nullptr, "null argument");
  B2RL_REQUIRE(r->owned && r->device == h->device, "fill needs the ring created for this replay, on its device");
  B2RL_REQUIRE(slot >= 0 && slot < r->L.slots, "slot out of range");
  B2RL_REQUIRE(h->dedup == nullptr || h->n_fields < B2RL_MAX_FIELDS, "too many fields to serve");
  int64_t bytes[B2RL_MAX_FIELDS];
  const int n = served_fields(h, bytes);
  B2RL_REQUIRE(r->L.n_fields == n, "ring and replay have different fields");
  for (int f = 0; f < n; ++f)
    B2RL_REQUIRE(bytes[f] == r->L.field_bytes[f], "ring and replay have different fields");
  B2RL_REQUIRE(h->size > 0, "sampling from an empty replay");
  return b2rl_serve_slot_ptrs(r, slot, ptrs, nullptr);
}

// One CTA per SM (the shared-memory ring takes the SM).  Split by items: at most one CTA per copy item, and
// enough CTAs that no item range touches more than SERVE_THREADS draws (a range of at most SERVE_THREADS - 2
// draws' items starts and ends inside at most SERVE_THREADS draws).  Split by draws: at most SERVE_THREADS each.
static int64_t fill_grid(int sms, int64_t n, const BulkRows& P, bool by_items) {
  const int64_t work = by_items ? n * (P.n > 0 ? P.items_per_row : 1) : n;
  int64_t grid = sms < work ? sms : work;
  const int64_t min_grid = by_items ? (n + SERVE_THREADS - 3) / (SERVE_THREADS - 2)
                                    : (n + SERVE_THREADS - 1) / SERVE_THREADS;
  return grid < min_grid ? min_grid : grid;
}

extern "C" int b2rl_serve_fill(b2rl_replay* h, b2rl_serve_ring* r, int32_t slot, uint64_t seq, float beta,
                               const float* max_w_dev, void* stream) {
  void* ptrs[3 + B2RL_MAX_FIELDS];
  int rc = fill_slot_ptrs(h, r, slot, ptrs);
  if (rc != B2RL_OK) return rc;
  BulkRows P{};
  SmallFields small{};
  SmallRows rows{};
  int host_f[B2RL_MAX_FIELDS], host_o[B2RL_MAX_FIELDS], n_host = 0;
  int host_planes_o = -1, coded_planes_o = -1;
  for (int f = 0, o = 3; f < h->n_fields; ++f, ++o) {
    const int64_t b = h->field_bytes[f];
    if (h->on_host[f]) {         // copied after the draw, from the slot's idx, by the host-row gather (hostrows.cu)
      host_f[n_host] = f;
      host_o[n_host++] = o;
    } else if (h->dedup != nullptr && f == dedup_planes_field(h) && dedup_pool_on_host(h)) {
      host_planes_o = o;         // the strips of a host pool: likewise, by the host-plane gather (hostrows.cu)
    } else if (h->dedup != nullptr && f == dedup_planes_field(h) && dedup_pool_coded(h)) {
      coded_planes_o = o;        // the strips, or s and s', of a coded pool: decoded after the draw, from the slot's
      if (dedup_strip_frames(h) == 0) ++o;   // idx (dedup.cu)
    } else if (h->dedup != nullptr && f == dedup_planes_field(h)) {   // frames assembled from the frame pool
      const int32_t* planes = (const int32_t*)h->field[f];
      const int R = dedup_strip_frames(h);
      if (R > 0) {                                                     // the strips
        P.add_planes(dedup_pool(h), planes, R, 0, R, (uint8_t*)ptrs[o]);
      } else {                                                         // the s and s' stacks
        P.add_planes(dedup_pool(h), planes, 8, 0, 4, (uint8_t*)ptrs[o]);
        P.add_planes(dedup_pool(h), planes, 8, 4, 4, (uint8_t*)ptrs[++o]);
      }
    } else if (is_bulk_row(b)) {
      P.add(h->field[f], (uint8_t*)ptrs[o], b, 14336);   // the CHUNK of k_serve_fill's copy_rows
    } else if (b == 1 || b == 2 || b == 4 || b == 8) {
      small.src[small.n] = h->field[f];
      small.dst[small.n] = (uint8_t*)ptrs[o];
      small.bytes[small.n] = (int)b;
      small.n++;
    } else {
      rows.f[rows.n++] = SmallField{h->field[f], (uint8_t*)ptrs[o], b};
    }
  }
  DeviceGuard g(h->device);
  int sms = 0;
  B2RL_CUDA(sm_count(h->device, &sms));
  B2RL_CUDA(set_max_dynamic_smem<k_serve_fill<true>>(h->device, BULK_RING_BYTES));
  B2RL_CUDA(set_max_dynamic_smem<k_serve_fill<false>>(h->device, BULK_RING_BYTES));
  const int64_t n = r->L.batch;
  const bool by_items = n < sms;
  auto kernel = by_items ? k_serve_fill<true> : k_serve_fill<false>;
  kernel<<<(unsigned)fill_grid(sms, n, P, by_items), SERVE_THREADS, BULK_RING_BYTES, (cudaStream_t)stream>>>(
      h->tree, P, small, rows, h->rng_dev, n, h->capacity, h->n_valid_dev, beta, max_w_dev, (int64_t*)ptrs[1],
      (float*)ptrs[2], (uint64_t*)ptrs[0], seq, r->done_ticket);
  count_launch();
  B2RL_CHECK_LAUNCH();
  for (int i = 0; i < n_host; ++i) {
    rc = gather_host_rows(h, host_f[i], (const int64_t*)ptrs[1], n, (uint8_t*)ptrs[host_o[i]], (cudaStream_t)stream);
    if (rc != B2RL_OK) return rc;
  }
  if (host_planes_o >= 0)
    return gather_host_planes(h, (const int64_t*)ptrs[1], n, (uint8_t*)ptrs[host_planes_o], (cudaStream_t)stream);
  if (coded_planes_o >= 0)
    return gather_coded_planes(h, (const int64_t*)ptrs[1], n, (uint8_t*)ptrs[coded_planes_o],
                               dedup_strip_frames(h) == 0 ? (uint8_t*)ptrs[coded_planes_o + 1] : nullptr,
                               (cudaStream_t)stream);
  return B2RL_OK;
}

extern "C" int b2rl_serve_fill_uniform(b2rl_replay* h, b2rl_serve_ring* r, int32_t slot, uint64_t seq, int32_t steps,
                                       void* stream) {
  void* ptrs[3 + B2RL_MAX_FIELDS];
  int rc = fill_slot_ptrs(h, r, slot, ptrs);
  if (rc != B2RL_OK) return rc;
  B2RL_REQUIRE(steps >= 1, "steps must be >= 1");
  B2RL_REQUIRE(h->dedup == nullptr || dedup_rollout_stacks(h) > 0,
               "a frame-deduplicated replay serves prioritized minibatches, not rollouts");
  B2RL_REQUIRE(h->dedup == nullptr || dedup_rollout_stacks(h) == steps + 1,
               "the rollout frame pool holds steps + 1 frame stacks per rollout: steps does not match it");
  B2RL_REQUIRE(!h->any_on_host, "a replay with fields placed on the host serves prioritized minibatches only");
  const int64_t n = r->L.batch, size = h->size, cap = h->capacity;
  B2RL_REQUIRE(n <= size, "sample larger than population: the batch exceeds the stored records");
  B2RL_REQUIRE(size <= (1LL << 32), "a uniform fill draws from at most 2^32 records");
  const UniformDraw u = uniform_draw_over(size, h->head, cap);
  BulkRows P{};
  SmallFields small{};
  SmallRows rows{};
  uint8_t* coded_stacks = nullptr;
  for (int f = 0; f < h->n_fields; ++f) {
    const int64_t b = h->field_bytes[f];
    if (h->dedup != nullptr && f == dedup_planes_field(h) && dedup_pool_coded(h)) {
      coded_stacks = (uint8_t*)ptrs[3 + f];   // decoded after the draw, from the slot's idx (dedup.cu)
      continue;
    }
    if (h->dedup != nullptr && f == dedup_planes_field(h)) {   // the stacks assembled from the frame pool
      P.add_planes_time_major(dedup_pool(h), (const int32_t*)h->field[f], dedup_strip_frames(h), steps + 1,
                              (uint8_t*)ptrs[3 + f]);
      continue;
    }
    RolloutField kind;
    const char* bad = rollout_field(b, steps, kind);
    B2RL_REQUIRE(bad == nullptr, bad);
    if (kind == RolloutField::FRAMES) {
      P.add_time_major(h->field[f], (uint8_t*)ptrs[3 + f], b, steps + 1, UNIFORM_CHUNK);
    } else if (kind == RolloutField::STEPS) {
      rows.f[rows.n++] = SmallField{h->field[f], (uint8_t*)ptrs[3 + f], b};
    } else {                     // a batch-major scalar
      small.src[small.n] = h->field[f];
      small.dst[small.n] = (uint8_t*)ptrs[3 + f];
      small.bytes[small.n] = (int)b;
      small.n++;
    }
  }
  DeviceGuard g(h->device);
  int sms = 0;
  B2RL_CUDA(sm_count(h->device, &sms));
  B2RL_CUDA(set_max_dynamic_smem<k_serve_fill_uniform<true>>(h->device, BULK_RING_BYTES));
  B2RL_CUDA(set_max_dynamic_smem<k_serve_fill_uniform<false>>(h->device, BULK_RING_BYTES));
  const bool by_items = n < sms;
  auto kernel = by_items ? k_serve_fill_uniform<true> : k_serve_fill_uniform<false>;
  kernel<<<(unsigned)fill_grid(sms, n, P, by_items), SERVE_THREADS, BULK_RING_BYTES, (cudaStream_t)stream>>>(
      P, small, rows, h->rng_dev, n, u, (int64_t*)ptrs[1], (uint64_t*)ptrs[0], seq, r->done_ticket);
  count_launch();
  B2RL_CHECK_LAUNCH();
  if (coded_stacks != nullptr)
    return decode_rollouts_time_major(h, (const int64_t*)ptrs[1], n, coded_stacks, (cudaStream_t)stream);
  return B2RL_OK;
}

extern "C" int b2rl_serve_take(const b2rl_serve_ring* r, int32_t slot, void* dst_dev, void* stream) {
  B2RL_REQUIRE(r != nullptr && dst_dev != nullptr, "null argument");
  B2RL_REQUIRE(slot >= 0 && slot < r->L.slots, "slot out of range");
  DeviceGuard g(r->device);
  B2RL_CUDA(cudaMemcpyAsync(dst_dev, r->base + (int64_t)slot * r->L.slot_bytes, (size_t)r->L.slot_bytes,
                            cudaMemcpyDefault, (cudaStream_t)stream));
  return B2RL_OK;
}

extern "C" int b2rl_serve_bind(const void* slot_dev, const b2rl_serve_layout* layout, int64_t n,
                               uint64_t* header_out_dev, int64_t* idx_out_dev, float* w_out_dev,
                               void* const* fields_out_dev, void* const* table_out_dev, void* stream) {
  B2RL_REQUIRE(slot_dev != nullptr, "null slot");
  B2RL_REQUIRE(layout != nullptr, "null layout");
  B2RL_REQUIRE((uintptr_t)slot_dev % 16 == 0, "the slot base must be 16-byte aligned");
  B2RL_REQUIRE(layout->n_fields >= 0 && layout->n_fields <= B2RL_MAX_FIELDS, "n_fields out of range");
  B2RL_REQUIRE(layout->batch == n, "the slot's batch does not match n");
  B2RL_REQUIRE(header_out_dev && idx_out_dev && w_out_dev, "null header, idx or w buffer");
  const uint8_t* s = (const uint8_t*)slot_dev;
  BindJobs J{};
  int jobs = 0;
  J.copy[jobs++] = BindCopy{s, (uint8_t*)header_out_dev, 16};
  J.copy[jobs++] = BindCopy{s + layout->idx_off, (uint8_t*)idx_out_dev, 8 * n};
  J.copy[jobs++] = BindCopy{s + layout->w_off, (uint8_t*)w_out_dev, 4 * n};
  for (int f = 0; f < layout->n_fields; ++f) {
    void* field_out = fields_out_dev ? fields_out_dev[f] : nullptr;
    void* entry = table_out_dev ? table_out_dev[f] : nullptr;
    B2RL_REQUIRE(!(field_out && entry), "a field is either copied or bound in the frame table, not both");
    if (field_out) J.copy[jobs++] = BindCopy{s + layout->field_off[f], (uint8_t*)field_out, layout->field_bytes[f] * n};
    if (entry) {
      B2RL_REQUIRE((uintptr_t)entry % 8 == 0, "a frame table entry must be 8-byte aligned");
      J.addr[J.n_entries] = s + layout->field_off[f];
      J.entry[J.n_entries++] = (const uint8_t**)entry;
    }
  }
  k_serve_bind<<<jobs, 256, 0, (cudaStream_t)stream>>>(J);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_serve_put_update(b2rl_serve_ring* r, int32_t slot, uint64_t seq, const int64_t* idx_dev,
                                     const float* prio_dev, int64_t n, void* stream) {
  B2RL_REQUIRE(r != nullptr, "null ring");
  B2RL_REQUIRE(slot >= 0 && slot < r->L.slots, "slot out of range");
  B2RL_REQUIRE(n >= 0 && n <= r->L.batch, "n out of range (0..batch)");
  B2RL_REQUIRE(n == 0 || (idx_dev != nullptr && prio_dev != nullptr), "null idx/prio");
  void* u[3];
  int rc = b2rl_serve_slot_ptrs(r, slot, nullptr, u);
  if (rc != B2RL_OK) return rc;
  DeviceGuard g(r->device);
  k_serve_put_update<<<1, 256, 0, (cudaStream_t)stream>>>((uint64_t*)u[0], (int64_t*)u[1], (float*)u[2], idx_dev,
                                                          prio_dev, n, seq);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}
