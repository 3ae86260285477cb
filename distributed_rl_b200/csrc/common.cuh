// Shared declarations for libb2rl (sm_90a).  Built with -fmad=false so every
// fp32/fp64 operation is individually rounded, which is what makes the kernels
// bit-comparable with the numpy oracle (oracle/oracle.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>

#include "../../include/b2rl.h"

namespace b2rl {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define B2RL_CUDA(call)                                                              \
  do {                                                                               \
    cudaError_t e_ = (call);                                                         \
    if (e_ != cudaSuccess) {                                                         \
      b2rl::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
      return B2RL_ERR_CUDA;                                                          \
    }                                                                                \
  } while (0)

#define B2RL_CHECK_LAUNCH()                                                          \
  do {                                                                               \
    cudaError_t e_ = cudaGetLastError();                                             \
    if (e_ != cudaSuccess) {                                                         \
      b2rl::set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e_)); \
      return B2RL_ERR_CUDA;                                                          \
    }                                                                                \
  } while (0)

#define B2RL_REQUIRE(cond, msg)                                                      \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      b2rl::set_error("%s:%d invalid argument: %s", __FILE__, __LINE__, msg);        \
      return B2RL_ERR_INVALID;                                                       \
    }                                                                                \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    target = dev;
  }
  ~DeviceGuard() {
    if (prev >= 0 && prev != target) cudaSetDevice(prev);
  }
  int target = -1;
};

// Multiprocessor count of device `dev`, queried once per device.
inline cudaError_t sm_count(int dev, int* out) {
  static int sms[64] = {0};
  if (!sms[dev & 63]) {
    const cudaError_t e = cudaDeviceGetAttribute(&sms[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
  }
  *out = sms[dev & 63];
  return cudaSuccess;
}

// Lets kernel K use `bytes` of dynamic shared memory on device `dev` (beyond the default 48 KiB); the attribute
// is set once per kernel and device.
template <auto K>
cudaError_t set_max_dynamic_smem(int dev, size_t bytes) {
  static bool done[64] = {false};
  if (done[dev & 63]) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) done[dev & 63] = true;
  return e;
}

// ---- device helpers --------------------------------------------------------

// x^e for fp32 operands: evaluated in fp64, rounded once ("powcr", DESIGN.md §3).
__device__ __forceinline__ float powcr(float x, float e) {
  return (float)pow((double)x, (double)e);
}

__host__ __device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

// Philox4x32-10 (Salmon et al. 2011), counter = (ctr_lo, ctr_hi, 0, 0), key = seed.
__host__ __device__ __forceinline__ void philox4x32_10(uint64_t ctr, uint64_t seed, uint32_t out[4]) {
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0u, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53U * c0;
    uint64_t p1 = (uint64_t)0xCD9E8D57U * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9U; k1 += 0xBB67AE85U;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// 53-bit uniform in [0,1) from one Philox block: (x & (2^53-1)) * 2^-53 (the
// reference's CPU generator is mt19937 with the same 53-bit mask construction).
__host__ __device__ __forceinline__ double philox_u01(uint64_t seed, uint64_t ctr) {
  uint32_t r[4];
  philox4x32_10(ctr, seed, r);
  uint64_t x = ((uint64_t)r[1] << 32) | r[0];
  return (double)(x & ((1ULL << 53) - 1)) * (1.0 / 9007199254740992.0);
}

// The slot a sampled index reads: indices outside [0, capacity) are clamped to the nearest slot.
__host__ __device__ __forceinline__ int64_t clamp_row(int64_t r, int64_t capacity) {
  return r < 0 ? 0 : (r >= capacity ? capacity - 1 : r);
}

}  // namespace b2rl

// The sum-tree as the kernels see it (tree.cu): a binary tree of depth `levels` stored sparsely — every 4th
// level only.  Stored level 0 = leaves (fp32 priorities, 0 = empty slot); stored level k (1 <= k < G) = binary
// depth levels-4k as fp64 sums + fp32 mins over valid leaves; stored level G = the root.  The levels in between
// are recomputed in registers with the binary tree's own pairwise association (bit-identical values).
constexpr int B2RL_TREE_MAX_GROUPS = 8;   // levels <= 32
struct TreeView {
  float* leaf;                              // [cap2]
  double* sum;                              // stored level k at sum + off[k]
  float* minv;                              // stored level k at minv + off[k]
  int64_t off[B2RL_TREE_MAX_GROUPS + 1];    // off[0] unused
  int64_t cap2;                             // leaves = 2^levels >= max(capacity, 2)
  int levels;
  int G;                                    // ceil(levels / 4) stored internal levels
  int top_bits;                             // binary levels spanned by the top group: levels - 4(G-1), in 1..4
};

struct b2rl_replay;
namespace b2rl {
// Stream-ordered publication of the host-side `size` to n_valid_dev (tree.cu).
int publish_size(b2rl_replay* h, cudaStream_t st);
// Record i of fields_src -> ring slot (start + i) % capacity; a NULL field is skipped (gather.cu).  Call
// check_host_sources first: a host field's source must be device or pinned host memory.
int check_host_sources(const b2rl_replay* h, const void* const* fields_src);
int copy_ring_range(b2rl_replay* h, const void* const* fields_src, int64_t start, int64_t n, cudaStream_t st);
// The n records at head become sampleable with the device priorities prios_dev; head moves past them (gather.cu).
int publish(b2rl_replay* h, const float* prios_dev, int64_t n, cudaStream_t st);
// Rows clamp_row(idx_dev[k]) of host field f -> dst_dev + k * field_bytes[f], k < n, through 16-byte loads of the
// mapped rows (hostrows.cu).  dst_dev 16-byte aligned.
int gather_host_rows(b2rl_replay* h, int f, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, cudaStream_t st);
// `bytes` from src (device or pinned host memory) into host field f from ring slot `slot` on, in stream order
// (hostrows.cu).
int copy_into_host_field(b2rl_replay* h, int f, int64_t slot, const uint8_t* src, int64_t bytes, cudaStream_t st);
struct DedupState;                       // the frame pool of a deduplicated replay (dedup.cu)
void dedup_free(b2rl_replay* h);
int dedup_planes_field(const b2rl_replay* h);
const uint8_t* dedup_pool(const b2rl_replay* h);  // the address kernels use (a host pool's device alias)
int64_t dedup_pool_frames(const b2rl_replay* h);
bool dedup_pool_on_host(const b2rl_replay* h);     // b2rl_dedup_attach_strips_placed with pool_on_host
int dedup_strip_frames(const b2rl_replay* h);     // R of a strip handle (b2rl_dedup_attach_strips), else 0
int dedup_rollout_stacks(const b2rl_replay* h);   // T + 1 of a rollout handle (b2rl_dedup_attach_rollouts), else 0
// The (n, R, 84, 84) strips of the sampled slots clamp_row(idx_dev[k]) of a strip handle whose pool is on the host,
// assembled from the pool through 16-byte loads of its mapped frames (hostrows.cu).  dst_dev 16-byte aligned.
int gather_host_planes(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, cudaStream_t st);
bool dedup_pool_coded(const b2rl_replay* h);      // b2rl_dedup_attach_strips_coded, _coded: frames encoded in a unit ring
// The frames of the sampled slots clamp_row(idx_dev[k]) of a handle whose pool is coded, decoded from the pool
// (dedup.cu): a strip handle's (n, R, 84, 84) strips into dst_dev (dst2_dev NULL), an Ape-X handle's s and s' stacks
// into dst_dev and dst2_dev (either may be NULL).  Outputs 16-byte aligned.
int gather_coded_planes(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, uint8_t* dst2_dev,
                        cudaStream_t st);
// The T + 1 stacks of the sampled slots clamp_row(idx_dev[k]) of a coded rollout handle, decoded time-major: stack t
// of draw k into row t * n + k of dst_dev, as b2rl_serve_fill_uniform lays out a slot's `state` (dedup.cu).  dst_dev
// 16-byte aligned.
int decode_rollouts_time_major(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, cudaStream_t st);
}  // namespace b2rl

// The opaque handle.
struct b2rl_replay {
  int device = 0;
  int64_t capacity = 0;   // requested slots
  int64_t cap2 = 0;       // tree leaves = 2^levels >= max(capacity, 2)
  int levels = 0;
  int n_fields = 0;
  int64_t field_bytes[B2RL_MAX_FIELDS] = {0};
  uint8_t* field[B2RL_MAX_FIELDS] = {nullptr};      // the address kernels use: device memory, or the device alias of
                                                    // a host field's pinned rows
  uint8_t* host_field[B2RL_MAX_FIELDS] = {nullptr}; // b2rl_replay_create_placed: the host address of a host field
  bool on_host[B2RL_MAX_FIELDS] = {false};
  bool any_on_host = false;
  TreeView tree = {};         // leaves + sparse fp64 levels (owned: tree.leaf, tree.sum, tree.minv)
  uint32_t* tag = nullptr;    // [cap2]   last-writer tags of the large scattered update, self-cleaning
  int64_t* scratch_idx = nullptr;  // [capacity] ring indices for push/evict
  float* scratch_val = nullptr;    // [capacity]
  uint64_t* rng_dev = nullptr;     // [3] device-resident Philox stream {seed, counter, ticket}
  unsigned int* build_ticket = nullptr;   // [1] last-CTA-done counter of the bulk build, self re-arming
  float* n_valid_dev = nullptr;    // [1] (float)size, rewritten in stream order whenever size changes: the
                                   //     sampling / stats kernels read it, so a captured graph never bakes it in
  int64_t size = 0;       // valid slots
  int64_t head = 0;       // next slot to write
  int64_t reserved = 0;   // slots zeroed by b2rl_replay_reserve and not yet committed
  // b2rl_replay_ingest_pipelined: library-owned copy stream + events, device staging of the pending priorities
  cudaStream_t ingest_stream = nullptr;
  cudaEvent_t ev_reserved = nullptr, ev_copied = nullptr;
  float* pipe_prios = nullptr;
  int64_t pipe_cap = 0;   // floats allocated at pipe_prios
  int64_t pipe_n = 0;     // records of the batch whose copy is in flight (0: none)
  b2rl::DedupState* dedup = nullptr;   // b2rl_dedup_attach: frame pool, key table, insertion marks
};
