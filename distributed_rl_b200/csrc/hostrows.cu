// Replay fields placed in pinned, mapped host memory (b2rl_replay_create_placed): the sampled-row gather over PCIe
// and the stream-ordered ingest into host rows.  The same gather for the frames of a strip handle whose frame pool is
// on the host (b2rl_dedup_attach_strips_placed): each sampled slot's R pool frames, scattered over the pool.
//
// A host field is never read by the TMA row copy of bulk_rows.cuh: whether bulk async copies read mapped host memory
// has not been established, so the rows travel through plain 16-byte loads of the mapped pointer.  PCIe latency is
// long (about a microsecond), so each thread keeps HOST_ROWS_UNROLL independent loads in flight before it stores
// any of them, and a few CTAs (B2RL_HOST_GATHER_CTAS, default HOST_GATHER_CTAS) are enough to fill the link: the
// copy leaves the rest of the GPU to the learner step.
#include "bulk_rows.cuh"

#include <stdlib.h>

namespace b2rl {

constexpr int HOST_ROWS_THREADS = 256;
constexpr int HOST_ROWS_UNROLL = 8;       // 16-byte loads in flight per thread
constexpr int HOST_GATHER_CTAS = 8;       // the fewest at the plateau of the B2RL_HOST_GATHER_CTAS sweep (§4.17)

// dst[k] = src row clamp_row(idx[k]) for k < n, rows of row_vecs 16-byte units; the n * row_vecs units are dealt out
// grid-stride, so consecutive threads read consecutive units of a row.
__global__ void __launch_bounds__(HOST_ROWS_THREADS)
k_gather_host_rows(const int4* __restrict__ src, int4* __restrict__ dst, int64_t row_vecs,
                   const int64_t* __restrict__ idx, int64_t n, int64_t capacity) {
  const int64_t total = n * row_vecs;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < total; v0 += stride * HOST_ROWS_UNROLL) {
    int4 r[HOST_ROWS_UNROLL];
#pragma unroll
    for (int u = 0; u < HOST_ROWS_UNROLL; ++u) {
      const int64_t v = v0 + u * stride;
      if (v < total) {
        const int64_t k = v / row_vecs;
        r[u] = __ldcg(src + clamp_row(idx[k], capacity) * row_vecs + (v - k * row_vecs));
      }
    }
#pragma unroll
    for (int u = 0; u < HOST_ROWS_UNROLL; ++u) {
      const int64_t v = v0 + u * stride;
      if (v < total) dst[v] = r[u];
    }
  }
}

// The frame-pool form of k_gather_host_rows, for a strip handle whose pool is on the host: dst row k (R frames of
// PLANE_BYTES) = the frames of slot clamp_row(idx[k]), frame j being pool frame planes[R slot + j] % F.  The n R frames'
// 16-byte units are dealt out grid-stride the same way, so a warp reads consecutive units of one frame.
__global__ void __launch_bounds__(HOST_ROWS_THREADS)
k_gather_host_planes(const int4* __restrict__ pool, int4* __restrict__ dst, const int32_t* __restrict__ planes,
                     int32_t R, int64_t F, const int64_t* __restrict__ idx, int64_t n, int64_t capacity) {
  constexpr int64_t FRAME_VECS = PLANE_BYTES / 16;   // 441
  const int64_t total = n * R * FRAME_VECS;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < total; v0 += stride * HOST_ROWS_UNROLL) {
    int4 r[HOST_ROWS_UNROLL];
#pragma unroll
    for (int u = 0; u < HOST_ROWS_UNROLL; ++u) {
      const int64_t v = v0 + u * stride;
      if (v < total) {
        const int64_t fr = v / FRAME_VECS;   // frame fr - k R of draw k
        const int64_t k = fr / R;
        const int64_t id = planes[R * clamp_row(idx[k], capacity) + (fr - k * R)];
        r[u] = __ldcg(pool + (id % F) * FRAME_VECS + (v - fr * FRAME_VECS));
      }
    }
#pragma unroll
    for (int u = 0; u < HOST_ROWS_UNROLL; ++u) {
      const int64_t v = v0 + u * stride;
      if (v < total) dst[v] = r[u];
    }
  }
}

// bytes from src to dst, both addressable by the device (here: a pinned host source into a host field's rows).
__global__ void __launch_bounds__(HOST_ROWS_THREADS)
k_copy_to_host_rows(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int64_t bytes) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if ((((uintptr_t)src | (uintptr_t)dst | (uintptr_t)bytes) & 15) == 0) {
    const int4* s = reinterpret_cast<const int4*>(src);
    int4* d = reinterpret_cast<int4*>(dst);
    const int64_t nv = bytes >> 4;
    for (int64_t v0 = t0; v0 < nv; v0 += stride * HOST_ROWS_UNROLL) {
      int4 r[HOST_ROWS_UNROLL];
#pragma unroll
      for (int u = 0; u < HOST_ROWS_UNROLL; ++u)
        if (v0 + u * stride < nv) r[u] = __ldcg(s + v0 + u * stride);
#pragma unroll
      for (int u = 0; u < HOST_ROWS_UNROLL; ++u)
        if (v0 + u * stride < nv) d[v0 + u * stride] = r[u];
    }
  } else {
    for (int64_t b = t0; b < bytes; b += stride) dst[b] = src[b];
  }
}

// CTAs of the host-row copies: B2RL_HOST_GATHER_CTAS when set (read at every call, so a sweep can change it between
// launches), else HOST_GATHER_CTAS; at most one per SM and no more than the work needs.
static int host_ctas(int dev, int64_t vecs) {
  int ctas = HOST_GATHER_CTAS;
  if (const char* e = getenv("B2RL_HOST_GATHER_CTAS")) ctas = atoi(e);
  int sms = 132;
  if (sm_count(dev, &sms) != cudaSuccess) cudaGetLastError();
  if (ctas > sms) ctas = sms;
  const int64_t need = (vecs + HOST_ROWS_THREADS - 1) / HOST_ROWS_THREADS;
  if (ctas > need) ctas = (int)need;
  return ctas < 1 ? 1 : ctas;
}

int gather_host_rows(b2rl_replay* h, int f, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, cudaStream_t st) {
  B2RL_REQUIRE((uintptr_t)dst_dev % 16 == 0, "the output rows of a host field must be 16-byte aligned");
  if (n == 0) return B2RL_OK;
  const int64_t row_vecs = h->field_bytes[f] / 16;
  k_gather_host_rows<<<host_ctas(h->device, n * row_vecs), HOST_ROWS_THREADS, 0, st>>>(
      reinterpret_cast<const int4*>(h->field[f]), reinterpret_cast<int4*>(dst_dev), row_vecs, idx_dev, n,
      h->capacity);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

int gather_host_planes(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, cudaStream_t st) {
  B2RL_REQUIRE((uintptr_t)dst_dev % 16 == 0, "frame strip outputs must be 16-byte aligned");
  if (n == 0) return B2RL_OK;
  const int R = dedup_strip_frames(h);
  k_gather_host_planes<<<host_ctas(h->device, n * R * (PLANE_BYTES / 16)), HOST_ROWS_THREADS, 0, st>>>(
      reinterpret_cast<const int4*>(dedup_pool(h)), reinterpret_cast<int4*>(dst_dev),
      (const int32_t*)h->field[dedup_planes_field(h)], R, dedup_pool_frames(h), idx_dev, n, h->capacity);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

// A host field's rows are written in stream order only: cudaMemcpyAsync from device memory, the copy kernel from
// pinned host memory.  cudaMemcpyAsync from host to host memory runs synchronously with the host, outside stream
// order: it could overwrite a slot a queued step has sampled and not yet read, so pageable sources are refused.
int check_host_sources(const b2rl_replay* h, const void* const* fields_src) {
  if (!h->any_on_host || fields_src == nullptr) return B2RL_OK;
  for (int f = 0; f < h->n_fields; ++f) {
    if (!h->on_host[f] || fields_src[f] == nullptr) continue;
    cudaPointerAttributes a{};
    B2RL_CUDA(cudaPointerGetAttributes(&a, fields_src[f]));
    B2RL_REQUIRE(a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged ||
                     (a.type == cudaMemoryTypeHost && a.devicePointer != nullptr),
                 "a field placed on the host takes its rows from device or pinned host memory, not pageable memory");
  }
  return B2RL_OK;
}

int copy_into_host_field(b2rl_replay* h, int f, int64_t slot, const uint8_t* src, int64_t bytes, cudaStream_t st) {
  if (bytes == 0) return B2RL_OK;
  cudaPointerAttributes a{};
  B2RL_CUDA(cudaPointerGetAttributes(&a, src));
  if (a.type == cudaMemoryTypeHost) {
    const uint8_t* s = (const uint8_t*)a.devicePointer;
    B2RL_REQUIRE(s != nullptr, "pinned host rows not mapped into the device's address space");
    k_copy_to_host_rows<<<host_ctas(h->device, (bytes + 15) / 16), HOST_ROWS_THREADS, 0, st>>>(
        s, h->field[f] + slot * h->field_bytes[f], bytes);
    count_launch();
    B2RL_CHECK_LAUNCH();
    return B2RL_OK;
  }
  B2RL_REQUIRE(a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged,
               "a field placed on the host takes its rows from device or pinned host memory, not pageable memory");
  B2RL_CUDA(cudaMemcpyAsync(h->host_field[f] + slot * h->field_bytes[f], src, (size_t)bytes, cudaMemcpyDeviceToHost,
                            st));
  return B2RL_OK;
}

}  // namespace b2rl
