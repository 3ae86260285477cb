// Mean all-reduce of a SMALL gradient slice across the data-parallel learner ranks of one node, over NVLink /
// NVSwitch peer memory, as one kernel per rank.
//
// The reference has a single learner process and no collective at all (SURVEY.md §8e: replay-sharded data
// parallelism is new work).  Per step the ranks average two gradient slices: the dense heads' (12.9 MB, launched
// early from the weight-gradient lane, NCCL) and what is left when backward ends — the convolution stack's
// 0.3 MB.  That second one sits on the critical path between backward and the optimizer, and is latency-bound: an
// NCCL all-reduce of it is a whole collective launch for little data (DESIGN.md §5).  Here every rank
//   0. copies its slice into its own symmetric staging buffer (parity = step & 1) and publishes a per-CTA flag
//      to every peer (st.release.sys after __threadfence_system),
//   1. waits for the same CTA's flag of every peer (ld.acquire.sys, bounded spin),
//   2. reads every rank's staged slice through the peer mapping, adds them IN RANK ORDER (so every rank forms the
//      bit-identical sum), scales by 1/world and writes its own gradient memory.
// No trailing barrier: a staging buffer is rewritten two steps later, and the heads' all-reduce of the step in
// between orders that write after every peer's read.  Flags only ever grow (epoch per CTA), nothing is reset.
#include "common.cuh"

namespace b2rl {
namespace peer {

constexpr int THREADS = 256;
constexpr int MAX_CTAS = 64;       // flag slots per (rank, peer)
constexpr int MAX_WORLD = 16;

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_peer(const float4* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

struct Params {
  const uint64_t* stage;    // [world] device pointers: rank r's staging buffer (2 x cap floats), peer-mapped
  const uint64_t* flags;    // [world] device pointers: rank r's flag pad (world x MAX_CTAS uint32), peer-mapped
  int32_t rank, world;
  int64_t cap;              // floats per staging parity
  int64_t n;                // floats to reduce (multiple of 4)
  float* data;              // this rank's slice: read, then overwritten with the mean
  uint32_t* epoch;          // [MAX_CTAS] per-CTA launch counters (device, private to this rank)
  uint32_t* error;          // set to 1 if a peer's flag did not arrive within the spin bound
};

__global__ void __launch_bounds__(THREADS)
k_peer_allreduce_mean(const __grid_constant__ Params P) {
  __shared__ uint32_t s_epoch;
  __shared__ const float4* s_src[MAX_WORLD];
  const int c = blockIdx.x, G = gridDim.x;
  if (threadIdx.x == 0) s_epoch = P.epoch[c] + 1u;
  __syncthreads();
  const uint32_t e = s_epoch;
  const int64_t quads = P.n >> 2;
  const int64_t q0 = quads * c / G, q1 = quads * (c + 1) / G;     // this CTA's float4 range
  float4* mine = reinterpret_cast<float4*>(P.stage[P.rank]) + (int64_t)(e & 1u) * (P.cap >> 2);
  float4* data = reinterpret_cast<float4*>(P.data);
  // 0. stage my slice where the peers can read it
  for (int64_t q = q0 + threadIdx.x; q < q1; q += THREADS) mine[q] = data[q];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < P.world) {
    const int p = threadIdx.x;
    s_src[p] = reinterpret_cast<const float4*>(P.stage[p]) + (int64_t)(e & 1u) * (P.cap >> 2);
    if (p != P.rank) {
      st_release_sys(reinterpret_cast<uint32_t*>(P.flags[p]) + P.rank * MAX_CTAS + c, e);
      // 1. wait for peer p's slice c of this step (bounded: ~2 s of polling, then flag the error and go on)
      const uint32_t* f = reinterpret_cast<const uint32_t*>(P.flags[P.rank]) + p * MAX_CTAS + c;
      long long spins = 0;
      while ((int32_t)(ld_acquire_sys(f) - e) < 0) {
        if (++spins > (1LL << 26)) { *P.error = 1u; break; }
        __nanosleep(20);
      }
    }
  }
  __syncthreads();
  // 2. sum in rank order (identical on every rank), scale, write my gradients
  const float inv = 1.0f / (float)P.world;
  for (int64_t q = q0 + threadIdx.x; q < q1; q += THREADS) {
    float4 a = ld_peer(s_src[0] + q);
    for (int p = 1; p < P.world; ++p) {
      const float4 b = ld_peer(s_src[p] + q);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    data[q] = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
  }
  if (threadIdx.x == 0) P.epoch[c] = e;
}


// ---- the LARGE slice (the dense heads' 12.9 MB): reduce-scatter + all-gather in one kernel ----------------------
// NCCL runs this as RING_LL on one NVSwitch node,
// which at 8 ranks ends only when backward does, so the heads' optimizer step behind it lands on the critical path.
// Here the gradient bucket itself is symmetric memory, and every rank r
//   1. publishes "my gradients are final" (per-CTA flag) and waits for the same flag of every peer,
//   2. reduces ITS 1/world slice: reads that slice of every rank's bucket through the peer mapping, adds in rank
//      order, scales, writes the result into its own bucket AND into its symmetric result buffer R (parity = step & 1),
//   3. publishes "R is ready", then copies every peer's R into the matching slice of its own bucket as each arrives.
// Each slice is reduced exactly once (by its owner), so all ranks end with bit-identical gradients.  A peer reads
// slice q of my bucket only in ITS step 2 and my R only in its step 3; I overwrite slice q only after R_q is
// published (i.e. after rank q has read it), and R is rewritten two steps later — no trailing barrier.
constexpr int BIG_THREADS = 512;

struct BigParams {
  const uint64_t* bucket;   // [world] device pointers: rank r's gradient bucket (peer-mapped), element 0 = slice start
  const uint64_t* result;   // [world] device pointers: rank r's R buffer (2 x slice_floats), peer-mapped
  const uint64_t* flags;    // [world] device pointers: rank r's flag pad: [2 phases][world][MAX_CTAS] uint32
  int32_t rank, world;
  int64_t n;                // floats (multiple of 4)
  int64_t slice;            // floats per rank slice (multiple of 4): rank r owns [r*slice, min((r+1)*slice, n))
  uint32_t* epoch;          // [MAX_CTAS]
  uint32_t* error;
};

__device__ __forceinline__ bool wait_flag(const uint32_t* f, uint32_t e, uint32_t* err) {
  long long spins = 0;
  while ((int32_t)(ld_acquire_sys(f) - e) < 0) {
    if (++spins > (1LL << 26)) { *err = 1u; return false; }
    __nanosleep(20);
  }
  return true;
}

__global__ void __launch_bounds__(BIG_THREADS)
k_peer_allreduce_big(const __grid_constant__ BigParams P) {
  __shared__ uint32_t s_epoch;
  __shared__ const float4* s_in[MAX_WORLD];
  const int c = blockIdx.x, G = gridDim.x, W = P.world, r = P.rank;
  if (threadIdx.x == 0) s_epoch = P.epoch[c] + 1u;
  __syncthreads();
  const uint32_t e = s_epoch;
  const int64_t sq = P.slice >> 2;                                   // float4 per slice
  uint32_t* my_flags = reinterpret_cast<uint32_t*>(P.flags[r]);
  // 1. my gradients are final (they were written by earlier kernels on this stream): tell every peer, wait for all
  __threadfence_system();
  if (threadIdx.x < W) {
    const int p = threadIdx.x;
    s_in[p] = reinterpret_cast<const float4*>(P.bucket[p]);
    if (p != r) {
      st_release_sys(reinterpret_cast<uint32_t*>(P.flags[p]) + (0 * W + r) * MAX_CTAS + c, e);
      wait_flag(my_flags + (0 * W + p) * MAX_CTAS + c, e, P.error);
    }
  }
  __syncthreads();
  // 2. reduce my slice (this CTA's share of it)
  const int64_t lo = (int64_t)r * sq, hi_all = P.n >> 2;
  const int64_t len = max((int64_t)0, min(sq, hi_all - lo));         // float4 in my slice (the last slice may be short)
  const int64_t q0 = len * c / G, q1 = len * (c + 1) / G;
  float4* my_bucket = reinterpret_cast<float4*>(P.bucket[r]);
  float4* my_R = reinterpret_cast<float4*>(P.result[r]) + (int64_t)(e & 1u) * sq;
  const float inv = 1.0f / (float)W;
  for (int64_t q = q0 + threadIdx.x; q < q1; q += 2 * BIG_THREADS) {
    const int64_t qb = q + BIG_THREADS;
    const bool two = qb < q1;
    float4 a = ld_peer(s_in[0] + lo + q), b = two ? ld_peer(s_in[0] + lo + qb) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = 1; p < W; ++p) {
      const float4 x = ld_peer(s_in[p] + lo + q);
      const float4 y = two ? ld_peer(s_in[p] + lo + qb) : make_float4(0.f, 0.f, 0.f, 0.f);
      a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
      b.x += y.x; b.y += y.y; b.z += y.z; b.w += y.w;
    }
    a = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
    my_R[q] = a;
    my_bucket[lo + q] = a;
    if (two) {
      b = make_float4(b.x * inv, b.y * inv, b.z * inv, b.w * inv);
      my_R[qb] = b;
      my_bucket[lo + qb] = b;
    }
  }
  __threadfence_system();
  __syncthreads();
  // 3. my R share is ready: tell every peer; then gather every peer's share as it arrives (start at my right
  //    neighbour so that the ranks do not all pull from the same GPU at once)
  if (threadIdx.x < W && threadIdx.x != r)
    st_release_sys(reinterpret_cast<uint32_t*>(P.flags[threadIdx.x]) + (1 * W + r) * MAX_CTAS + c, e);
  for (int k = 1; k < W; ++k) {
    const int p = (r + k) % W;
    if (threadIdx.x == 0) wait_flag(my_flags + (1 * W + p) * MAX_CTAS + c, e, P.error);
    __syncthreads();
    const int64_t plo = (int64_t)p * sq;
    const int64_t plen = max((int64_t)0, min(sq, hi_all - plo));
    const int64_t p0 = plen * c / G, p1 = plen * (c + 1) / G;
    const float4* R = reinterpret_cast<const float4*>(P.result[p]) + (int64_t)(e & 1u) * sq;
    for (int64_t q = p0 + threadIdx.x; q < p1; q += BIG_THREADS) my_bucket[plo + q] = ld_peer(R + q);
  }
  if (threadIdx.x == 0) P.epoch[c] = e;
}

}  // namespace peer
}  // namespace b2rl

using namespace b2rl;

extern "C" int32_t b2rl_peer_allreduce_max_ctas(void) { return peer::MAX_CTAS; }

extern "C" int b2rl_peer_allreduce_mean(const uint64_t* stage_ptrs_dev, const uint64_t* flag_ptrs_dev, int32_t rank,
                                        int32_t world, int64_t stage_cap_floats, float* data_dev, int64_t n,
                                        uint32_t* epoch_dev, uint32_t* error_dev, void* stream) {
  B2RL_REQUIRE(stage_ptrs_dev && flag_ptrs_dev && data_dev && epoch_dev && error_dev, "null argument");
  B2RL_REQUIRE(world >= 2 && world <= peer::MAX_WORLD && rank >= 0 && rank < world, "2..16 ranks");
  B2RL_REQUIRE(n >= 4 && (n % 4) == 0 && n <= stage_cap_floats && (stage_cap_floats % 4) == 0,
               "n must be a multiple of 4 within the staging capacity");
  B2RL_REQUIRE(((uintptr_t)data_dev % 16) == 0, "data must be 16-byte aligned");
  peer::Params P{stage_ptrs_dev, flag_ptrs_dev, rank, world, stage_cap_floats, n, data_dev, epoch_dev, error_dev};
  const int64_t quads = n >> 2;
  int64_t g = (quads + 4 * peer::THREADS - 1) / (4 * peer::THREADS);     // ~4 float4 per thread
  if (g < 1) g = 1;
  if (g > peer::MAX_CTAS) g = peer::MAX_CTAS;
  peer::k_peer_allreduce_mean<<<(unsigned)g, peer::THREADS, 0, (cudaStream_t)stream>>>(P);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_peer_allreduce_mean_big(const uint64_t* bucket_ptrs_dev, const uint64_t* result_ptrs_dev,
                                            const uint64_t* flag_ptrs_dev, int32_t rank, int32_t world, int64_t n,
                                            int64_t slice_floats, int32_t ctas, uint32_t* epoch_dev,
                                            uint32_t* error_dev, void* stream) {
  B2RL_REQUIRE(bucket_ptrs_dev && result_ptrs_dev && flag_ptrs_dev && epoch_dev && error_dev, "null argument");
  B2RL_REQUIRE(world >= 2 && world <= peer::MAX_WORLD && rank >= 0 && rank < world, "2..16 ranks");
  B2RL_REQUIRE(n >= 4 && (n % 4) == 0 && slice_floats >= 4 && (slice_floats % 4) == 0 &&
                   slice_floats * world >= n, "n and the slice must be multiples of 4 and the slices must cover n");
  B2RL_REQUIRE(ctas >= 1 && ctas <= peer::MAX_CTAS, "1..64 CTAs");
  peer::BigParams P{bucket_ptrs_dev, result_ptrs_dev, flag_ptrs_dev, rank, world, n, slice_floats, epoch_dev, error_dev};
  peer::k_peer_allreduce_big<<<(unsigned)ctas, peer::BIG_THREADS, 0, (cudaStream_t)stream>>>(P);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}
