// Device-resident sum-tree: bulk build, proportional sampling + IS weights,
// deterministic batched priority update, stats.
//
// Semantics follow the reference's own sum-tree (baseline/sumtree.py) exactly:
// fp64 nodes, node = fl64(left + right) (Node._reduce :21-27), descent
// `pos < left ? left : (pos -= left, right)` (Node._find :53-62).  The flat
// fp32 store the live learners use (baseline/PER.py) agrees with it whenever
// its own fp32 cumulative sums are exact (tests/golden/tree.npz, dyadic cases).
//
// Layout (DESIGN.md §3/§4, round 2): the binary tree is stored SPARSELY — only
// every 4th level is materialised.  Stored level 0 = the leaves as fp32 (the
// priorities themselves; (double)p is exact), stored level k = the binary
// tree's depth L-4k as fp64 sums (+ fp32 mins), the last stored level is the
// root.  The three levels in between are recomputed in registers from the 16
// children with the SAME pairwise association ((c0+c1)+(c2+c3))+..., so every
// value a binary tree would hold — and therefore every comparison of the
// reference's descent — is reproduced bit for bit.  Effects:
//   * a descent is ceil(L/4) dependent 128-byte loads instead of L (5 for 2^20)
//   * a path refresh is ceil(L/4) line reads + 8-byte writes, no atomics: the
//     recompute is a pure function of final children, so duplicate recomputes
//     by several threads are benign and only level barriers are needed
//   * the tree costs 4N + N/15*12 bytes instead of 32N, and a bulk build moves
//     ~8.8N bytes (4N read, 4N leaf copy, 0.75N nodes) for 8N algorithmic
#include "common.cuh"
#include "tree.cuh"

#include <math.h>
#include <stdlib.h>

namespace b2rl {

// ----------------------------------------------------------------------------
// 16-wide group arithmetic (ld4f / load_child_sums / descend16 live in tree.cuh)
// ----------------------------------------------------------------------------
template <bool CG>
__device__ __forceinline__ float load_child_min(const TreeView& t, int k, int64_t node) {
  const int bits = (k == t.G) ? t.top_bits : 4;
  const float* p = (k == 1) ? t.leaf + (node << bits) : t.minv + t.off[k - 1] + (node << bits);
  float m = INFINITY;
  if (bits == 4) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = ld4f<CG>(p + 4 * q);
      if (k == 1) {   // leaves: only valid (p > 0) slots take part in the min
        m = fminf(m, v.x > 0.0f ? v.x : INFINITY); m = fminf(m, v.y > 0.0f ? v.y : INFINITY);
        m = fminf(m, v.z > 0.0f ? v.z : INFINITY); m = fminf(m, v.w > 0.0f ? v.w : INFINITY);
      } else {
        m = fminf(fminf(m, v.x), fminf(v.y, fminf(v.z, v.w)));
      }
    }
  } else {
    for (int i = 0; i < (1 << bits); ++i) {
      const float v = CG ? __ldcg(p + i) : p[i];
      m = fminf(m, (k == 1 && !(v > 0.0f)) ? INFINITY : v);
    }
  }
  return m;
}

// ((c0+c1)+(c2+c3)) + ... : the value the binary tree stores 4 levels up.
__device__ __forceinline__ double pairwise16(const double c[16]) {
  double s1[8], s2[4];
#pragma unroll
  for (int i = 0; i < 8; ++i) s1[i] = c[2 * i] + c[2 * i + 1];
#pragma unroll
  for (int i = 0; i < 4; ++i) s2[i] = s1[2 * i] + s1[2 * i + 1];
  return (s2[0] + s2[1]) + (s2[2] + s2[3]);
}

template <bool CG>
__device__ __forceinline__ void recompute_node(const TreeView& t, int k, int64_t node) {
  double c[16];
  load_child_sums<CG>(t, k, node, c);
  const float m = load_child_min<CG>(t, k, node);
  t.sum[t.off[k] + node] = pairwise16(c);
  t.minv[t.off[k] + node] = m;
}

// ----------------------------------------------------------------------------
// Bulk build
// ----------------------------------------------------------------------------
constexpr int BUILD_THREADS = 256;
constexpr int BUILD_LEAVES = BUILD_THREADS * 16;   // 4096 leaves per CTA: stored levels 1..3 resolved in the CTA

// A CTA owns 4096 consecutive leaves.  Every thread moves four float4 (fully coalesced: a warp reads and writes
// 512 contiguous bytes per instruction, all four loads in flight before the first use); the four lanes that
// share a 16-leaf group fold their partial sums with two xor-shuffles — fp64 addition is commutative, so
// ((c0+c1)+(c2+c3)) + ... comes out bit-identical on all four lanes.  The CTA then folds its 256 level-1 nodes
// into 16 level-2 nodes and one level-3 node through shared memory.  Only levels below the top group (k < G)
// are produced here: their groups are full 16-wide by construction.
template <bool VEC>
__global__ void __launch_bounds__(BUILD_THREADS)
k_build_leaves(const __grid_constant__ TreeView t, const float* __restrict__ prios, int64_t n_valid, int fused_upto,
               unsigned int* __restrict__ ticket) {
  __shared__ double s_sum[BUILD_THREADS];
  __shared__ float s_min[BUILD_THREADS];
  __shared__ double s_sum2[16];
  __shared__ float s_min2[16];
  const int tid = threadIdx.x;
  const int64_t cta_base = (int64_t)blockIdx.x * BUILD_LEAVES;
  float4 v[4];
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int64_t base = cta_base + ((int64_t)it * BUILD_THREADS + tid) * 4;
    if (VEC && base + 4 <= n_valid) {
      v[it] = __ldcs(reinterpret_cast<const float4*>(prios + base));   // streamed once
    } else {
      v[it].x = (base + 0 < n_valid) ? prios[base + 0] : 0.0f;
      v[it].y = (base + 1 < n_valid) ? prios[base + 1] : 0.0f;
      v[it].z = (base + 2 < n_valid) ? prios[base + 2] : 0.0f;
      v[it].w = (base + 3 < n_valid) ? prios[base + 3] : 0.0f;
    }
  }
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int64_t base = cta_base + ((int64_t)it * BUILD_THREADS + tid) * 4;
    if (base + 4 <= t.cap2) {
      *reinterpret_cast<float4*>(t.leaf + base) = v[it];
    } else if (base < t.cap2) {          // cap2 == 2
      t.leaf[base] = v[it].x;
      t.leaf[base + 1] = v[it].y;
    }
    // quarter of a 16-leaf group -> whole group by two butterfly steps (all 32 lanes take part)
    double q = ((double)v[it].x + (double)v[it].y) + ((double)v[it].z + (double)v[it].w);
    float m = fminf(fminf(v[it].x > 0.0f ? v[it].x : INFINITY, v[it].y > 0.0f ? v[it].y : INFINITY),
                    fminf(v[it].z > 0.0f ? v[it].z : INFINITY, v[it].w > 0.0f ? v[it].w : INFINITY));
    q = q + __shfl_xor_sync(0xffffffffu, q, 1);
    m = fminf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    q = q + __shfl_xor_sync(0xffffffffu, q, 2);
    m = fminf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    if ((tid & 3) == 0) {
      s_sum[it * 64 + (tid >> 2)] = q;
      s_min[it * 64 + (tid >> 2)] = m;
      if (fused_upto >= 1 && base < t.cap2) {
        t.sum[t.off[1] + (base >> 4)] = q;
        t.minv[t.off[1] + (base >> 4)] = m;
      }
    }
  }
  if (fused_upto >= 2) {
    __syncthreads();
    if (tid < 16) {
      const int64_t node2 = (int64_t)blockIdx.x * 16 + tid;
      double c[16];
      float m2 = INFINITY;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        c[i] = s_sum[tid * 16 + i];
        m2 = fminf(m2, s_min[tid * 16 + i]);
      }
      const double val = pairwise16(c);
      if ((node2 << 8) < t.cap2) {
        t.sum[t.off[2] + node2] = val;
        t.minv[t.off[2] + node2] = m2;
      }
      s_sum2[tid] = val;
      s_min2[tid] = m2;
    }
    if (fused_upto >= 3) {
      __syncthreads();
      if (tid == 0) {
        double c[16];
        float m3 = INFINITY;
#pragma unroll
        for (int i = 0; i < 16; ++i) { c[i] = s_sum2[i]; m3 = fminf(m3, s_min2[i]); }
        t.sum[t.off[3] + blockIdx.x] = pairwise16(c);
        t.minv[t.off[3] + blockIdx.x] = m3;
      }
    }
  }
  // The LAST CTA to get here builds the remaining levels (<= cap2 / 65536 nodes on the widest of them; the
  // whole tree when it is small): no second launch.
  if (ticket == nullptr) return;     // two-launch variant: k_tree_top follows
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int prev = atomicAdd(ticket, 1u);
    s_last = (prev == gridDim.x - 1);
    if (s_last) *ticket = 0u;        // re-armed for the next build (graph replays included)
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int k = fused_upto + 1; k <= t.G; ++k) {
    const int64_t nk = (k == t.G) ? 1 : (t.cap2 >> (4 * k));
    for (int64_t node = tid; node < nk; node += BUILD_THREADS) recompute_node<true>(t, k, node);
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------
// Sampling + importance weights (+ optional fetch of the sampled slots' scalar fields)
// ----------------------------------------------------------------------------
constexpr int SAMPLE_THREADS = 128;

__global__ void __launch_bounds__(SAMPLE_THREADS)
k_tree_sample(const __grid_constant__ TreeView t, const double* __restrict__ u01, uint64_t seed, uint64_t rng_offset,
              const uint64_t* __restrict__ rng_state, int64_t n, const float* __restrict__ n_valid_dev, float beta,
              const float* __restrict__ max_w_ext, int64_t* __restrict__ idx_out,
              float* __restrict__ prob_out, float* __restrict__ w_out, SmallFields small) {
  const int64_t k = (int64_t)blockIdx.x * SAMPLE_THREADS + threadIdx.x;
  if (rng_state) rng_stream_take(const_cast<uint64_t*>(rng_state), n, seed, rng_offset);
  if (k >= n) return;
  const double u = u01 ? u01[k] : philox_u01(seed, rng_offset + (uint64_t)k);
  double root, picked;
  const int64_t j = tree_draw(t, u, root, picked);
  idx_out[k] = j;
  fetch_small(small, j, k);                 // scalar fields of the sampled slot (a, r, done)
  if (prob_out == nullptr && w_out == nullptr) return;
  const float s32 = (float)root;
  const float p = (float)picked;
  const float prob = __fdiv_rn(p, s32);
  if (prob_out) prob_out[k] = prob;
  if (w_out) w_out[k] = is_weight(t, s32, prob, n_valid_dev, beta, max_w_ext);
}

__global__ void k_rng_seed(uint64_t* __restrict__ rng_state, uint64_t seed, uint64_t ctr) {
  rng_state[0] = seed; rng_state[1] = ctr; rng_state[2] = 0;
}

__global__ void k_philox_uniforms(uint64_t seed, uint64_t off, int64_t n, double* __restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = philox_u01(seed, off + (uint64_t)k);
}

__global__ void k_set_n_valid(float* __restrict__ n_valid_dev, float v) { *n_valid_dev = v; }

__global__ void k_tree_stats(const __grid_constant__ TreeView t, const float* __restrict__ n_valid_dev, float beta,
                             double* __restrict__ out, float* __restrict__ max_w_out) {
  const float n_valid = *n_valid_dev;
  const double root = t.sum[t.off[t.G]];
  const float s32 = (float)root;
  const float mn = t.minv[t.off[t.G]];
  const float mw = powcr(__fmul_rn(n_valid, __fdiv_rn(mn, s32)), -beta);
  if (out) { out[0] = root; out[1] = (double)mn; out[2] = (double)mw; }
  if (max_w_out) *max_w_out = mw;
}

__global__ void k_tree_leaves(const __grid_constant__ TreeView t, int64_t start, int64_t n, float* __restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = t.leaf[start + k];
}

// ----------------------------------------------------------------------------
// Batched priority update — deterministic last-writer-wins, no fp atomics.
// Leaves are written by the winner of each slot; every stored level is then
// recomputed from its (final) children, level by level.  Several batch entries
// under one node recompute the same value — harmless, so no per-node ownership
// is needed, only a barrier per stored level (ceil(L/4) of them).
// ----------------------------------------------------------------------------
__device__ __forceinline__ int64_t upd_index(const int64_t* idx, int64_t ring_start, int64_t capacity,
                                             int64_t k) {
  if (idx) return idx[k];
  int64_t j = ring_start + k;
  return j >= capacity ? j - capacity : j;
}

__device__ __forceinline__ int64_t node_of(const TreeView& t, int k, int64_t leaf) {
  return (k == t.G) ? 0 : (leaf >> (4 * k));
}

// Small batch (n <= 512 per launch): ONE CTA.
//   0. slot ids -> shared memory, chained into a 1024-bucket hash table (atomicExch on the bucket head): the
//      last occurrence of a slot in the batch is its winner (baseline/PER.py:42) and is found by walking one
//      short chain (a linear scan of the batch cost 5.5 k cycles, this 0.9 k); winners write their leaves
//   1. stored levels 1..ks (the levels with more than US_SMEM_NODES nodes, plus the first one that fits): one
//      global round trip each — the node is recomputed from its 16 children by the first of the neighbouring
//      entries that share it (L1-cached loads: the CTA is the only writer, __syncthreads orders them)
//   2. level ks was preloaded into shared memory at kernel start and is patched with the new values; every
//      level above it is recomputed for ALL of its (<= 256) nodes from shared memory (rows padded to 17
//      entries: conflict-free) — no further global round trips, no contention on the few top nodes
// 2^20 leaves: 2 global round trips (65536- and 4096-node levels) + 3 shared-memory levels.
// (A variant with 16 lanes per node and shuffle butterflies was measured slower: 16 passes of shuffles cost
//  more issue slots than the 16-byte loads they saved.)
constexpr int US_THREADS = 512;
constexpr int US_SMEM_NODES = 4096;                         // level ks: up to 4096 nodes
constexpr int US_PAD_NODES = US_SMEM_NODES + US_SMEM_NODES / 16;   // rows of 16 children padded to 17
constexpr int US_TOP_NODES = 256 + 16 + 16 + 16 + 16;       // all nodes of the levels above ks, each level padded
constexpr int US_BUCKETS = 1024;
constexpr size_t US_SMEM_BYTES = (size_t)(US_PAD_NODES + US_TOP_NODES) * 12 + US_THREADS * 4 + US_BUCKETS * 4 + US_THREADS * 4;

__device__ __forceinline__ int us_pad(int i) { return i + (i >> 4); }

__global__ void __launch_bounds__(US_THREADS, 1)
k_update_small(const __grid_constant__ TreeView t, const int64_t* __restrict__ idx, int64_t ring_start,
               int64_t capacity, const float* __restrict__ vals, float const_val, int n, int ks,
               float* __restrict__ n_valid_dev, float n_valid_new, long long* __restrict__ probe) {
#define US_PROBE(i) do { if (probe != nullptr && threadIdx.x == 0) probe[i] = clock64(); } while (0)
  extern __shared__ __align__(16) unsigned char us_smem[];
  US_PROBE(0);
  double* s_sum = reinterpret_cast<double*>(us_smem);                     // level ks (padded rows)
  double* s_top = s_sum + US_PAD_NODES;                                   // levels > ks, packed (padded rows)
  float* s_min = reinterpret_cast<float*>(s_top + US_TOP_NODES);
  float* s_topm = s_min + US_PAD_NODES;
  int32_t* s_j = reinterpret_cast<int32_t*>(s_topm + US_TOP_NODES);
  int32_t* s_head = s_j + US_THREADS;
  int32_t* s_next = s_head + US_BUCKETS;
  const int tid = threadIdx.x;
  if (n_valid_dev != nullptr && tid == 0) *n_valid_dev = n_valid_new;   // ring size after this ingest step
  int32_t j = -1;
  if (tid < n) {
    const int64_t jj = upd_index(idx, ring_start, capacity, tid);
    if (jj >= 0 && jj < capacity) j = (int32_t)jj;    // out-of-range indices are ignored
  }
  s_j[tid] = j;
  s_head[tid] = -1; s_head[tid + US_THREADS] = -1;
  // preload stored level ks (old values; the touched entries are patched below)
  const int nks = (ks == t.G) ? 1 : (int)(t.cap2 >> (4 * ks));
  for (int i = tid; i < nks; i += US_THREADS) {
    s_sum[us_pad(i)] = t.sum[t.off[ks] + i];
    s_min[us_pad(i)] = t.minv[t.off[ks] + i];
  }
  const float myval = (j >= 0 && vals != nullptr) ? vals[tid] : const_val;
  __syncthreads();
  US_PROBE(1);
  const unsigned bucket = (unsigned)(lowbias32((uint32_t)j) & (US_BUCKETS - 1));
  if (idx != nullptr) {      // ring ranges have no duplicates
    if (j >= 0) s_next[tid] = atomicExch(s_head + bucket, tid);
    __syncthreads();
  }
  if (j >= 0) {
    bool dup = false;                                       // does a LATER entry name the same slot?
    if (idx != nullptr)
      for (int q = s_head[bucket]; q >= 0; q = s_next[q]) dup = dup || (q > tid && s_j[q] == j);
    if (!dup) t.leaf[j] = myval;
  }
  US_PROBE(2);
  __syncthreads();
  US_PROBE(3);
  for (int k = 1; k <= ks; ++k) {
    if (j >= 0) {
      const int64_t node = node_of(t, k, j);
      bool mine = true;               // neighbours under the same node leave the work to the first of them
      if (tid > 0) {
        const int32_t jp = s_j[tid - 1];
        if (jp >= 0 && node_of(t, k, jp) == node) mine = false;
      }
      if (mine) {
        double c[16];
        load_child_sums<false>(t, k, node, c);
        const float m = load_child_min<false>(t, k, node);
        const double v = pairwise16(c);
        t.sum[t.off[k] + node] = v;
        t.minv[t.off[k] + node] = m;
        if (k == ks) { s_sum[us_pad((int)node)] = v; s_min[us_pad((int)node)] = m; }
      }
    }
    __syncthreads();
    US_PROBE(3 + k);
  }
  // levels above ks: every node, children from shared memory
  const double* c_sum = s_sum;
  const float* c_min = s_min;
  int top_off = 0;
  for (int k = ks + 1; k <= t.G; ++k) {
    const int bits = (k == t.G) ? t.top_bits : 4;
    const int nk = (k == t.G) ? 1 : (int)(t.cap2 >> (4 * k));
    if (tid < nk) {
      double c[16];
      float m = INFINITY;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const bool in = i < (1 << bits);
        const int ci = us_pad((tid << bits) + i);           // children rows are padded: (tid*16+i) + tid
        c[i] = in ? c_sum[ci] : 0.0;
        m = fminf(m, in ? c_min[ci] : INFINITY);
      }
      const double v = pairwise16(c);
      s_top[top_off + us_pad(tid)] = v;
      s_topm[top_off + us_pad(tid)] = m;
      t.sum[t.off[k] + tid] = v;
      t.minv[t.off[k] + tid] = m;
    }
    __syncthreads();
    c_sum = s_top + top_off;
    c_min = s_topm + top_off;
    top_off += us_pad(nk) + 1;
  }
  US_PROBE(12);
#undef US_PROBE
}

// Stored levels k_first..G for ALL their nodes, one CTA, level-synchronous (the widest has <= 4096 nodes when
// called from the update path; the build path calls it with cap2 / 65536 nodes at most).
__global__ void __launch_bounds__(1024)
k_tree_top(const __grid_constant__ TreeView t, int k_first) {
  for (int k = k_first; k <= t.G; ++k) {
    const int64_t nk = (k == t.G) ? 1 : (t.cap2 >> (4 * k));
    // plain (L1-cached) loads: level k_first-1 was written by an earlier launch, the levels above by this CTA
    // itself before a __syncthreads — and no line of them was read earlier in this launch
    for (int64_t node = threadIdx.x; node < nk; node += blockDim.x) recompute_node<false>(t, k, node);
    __syncthreads();
  }
}

// One stored level, every node (used by the large update when the batch touches most of the level anyway).
__global__ void __launch_bounds__(256)
k_tree_level_all(const __grid_constant__ TreeView t, int k) {
  const int64_t nk = (k == t.G) ? 1 : (t.cap2 >> (4 * k));
  const int64_t node = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (node < nk) recompute_node<true>(t, k, node);
}

// Large scattered batch: tag -> write -> one launch per stored level.
constexpr int UPD_THREADS = 256;

__global__ void __launch_bounds__(UPD_THREADS)
k_update_tag(const int64_t* __restrict__ idx, int64_t capacity, int64_t n, uint32_t* __restrict__ tag) {
  const int64_t k = (int64_t)blockIdx.x * UPD_THREADS + threadIdx.x;
  if (k >= n) return;
  const int64_t j = idx[k];
  if (j < 0 || j >= capacity) return;
  atomicMax(tag + j, (uint32_t)(k + 1));     // integer atomics only: who is the last writer?
}

__global__ void __launch_bounds__(UPD_THREADS)
k_update_write(const __grid_constant__ TreeView t, const int64_t* __restrict__ idx, int64_t capacity, const float* __restrict__ vals,
               float const_val, int64_t n, uint32_t* __restrict__ tag) {
  const int64_t k = (int64_t)blockIdx.x * UPD_THREADS + threadIdx.x;
  if (k >= n) return;
  const int64_t j = idx[k];
  if (j < 0 || j >= capacity) return;
  if (tag[j] != (uint32_t)(k + 1)) return;   // a later k wrote the same slot
  t.leaf[j] = vals ? vals[k] : const_val;
  tag[j] = 0u;                                // self-clean: only the winner touches it here
}

__global__ void __launch_bounds__(UPD_THREADS)
k_update_level(const __grid_constant__ TreeView t, int k, const int64_t* __restrict__ idx, int64_t capacity, int64_t n) {
  const int64_t q = (int64_t)blockIdx.x * UPD_THREADS + threadIdx.x;
  if (q >= n) return;
  const int64_t j = idx[q];
  if (j < 0 || j >= capacity) return;
  recompute_node<true>(t, k, node_of(t, k, j));
}

// Large ring range [start, start+n) mod capacity (ingest / eviction): slots are distinct and contiguous,
// so leaves are written coalesced and each level touches ~n/16^k nodes: one thread per touched node.
__global__ void __launch_bounds__(UPD_THREADS)
k_update_range_write(const __grid_constant__ TreeView t, int64_t ring_start, int64_t capacity, const float* __restrict__ vals,
                     float const_val, int64_t n) {
  const int64_t k = (int64_t)blockIdx.x * UPD_THREADS + threadIdx.x;
  if (k >= n) return;
  t.leaf[upd_index(nullptr, ring_start, capacity, k)] = vals ? vals[k] : const_val;
}

__global__ void __launch_bounds__(UPD_THREADS)
k_update_range_level(const __grid_constant__ TreeView t, int k, int64_t a0, int64_t b0, int64_t a1, int64_t b1) {
  // segments [a0, b0) and [a1, b1) of leaf ids (the second is empty unless the ring wrapped)
  const int sh = 4 * k;
  const int64_t f0 = (k == t.G) ? 0 : (a0 >> sh), l0 = (k == t.G) ? 0 : ((b0 - 1) >> sh);
  const int64_t c0 = l0 - f0 + 1;
  const int64_t q = (int64_t)blockIdx.x * UPD_THREADS + threadIdx.x;
  if (q < c0) { recompute_node<true>(t, k, f0 + q); return; }
  if (b1 <= a1) return;
  const int64_t f1 = (k == t.G) ? 0 : (a1 >> sh), l1 = (k == t.G) ? 0 : ((b1 - 1) >> sh);
  if (q - c0 <= l1 - f1) recompute_node<true>(t, k, f1 + (q - c0));
}

}  // namespace b2rl

using namespace b2rl;

static inline unsigned grid_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

int b2rl::publish_size(b2rl_replay* h, cudaStream_t st) {
  k_set_n_valid<<<1, 1, 0, st>>>(h->n_valid_dev, (float)h->size);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

// idx_dev == nullptr means the ring range [ring_start, ring_start+n) (mod capacity);
// vals_dev == nullptr means the constant `const_val`.
int b2rl_tree_update_impl(b2rl_replay* h, const int64_t* idx_dev, int64_t ring_start,
                          const float* vals_dev, float const_val, int64_t n, cudaStream_t st,
                          bool publish_size_too) {
  if (n == 0) return publish_size_too ? publish_size(h, st) : B2RL_OK;
  const TreeView& t = h->tree;
  static int force_large = -1;
  if (force_large < 0) {
    const char* e = getenv("B2RL_UPDATE");
    force_large = (e && (e[0] == 'a' || e[0] == 'l')) ? 1 : 0;   // B2RL_UPDATE=large forces the multi-launch path
  }
  // first stored level that fits the small kernel's shared memory / the single-CTA top kernel
  int ks = 1;
  while (ks < t.G && (t.cap2 >> (4 * ks)) > US_SMEM_NODES) ++ks;
  if (!force_large && n <= US_THREADS) {      // (two chunked launches cost 21 us, the large path 14 us)
    static long long* probe = nullptr;
    static bool attr_set = false;
    if (!attr_set) {
      if (getenv("B2RL_TREE_PROBE")) cudaMalloc(&probe, 16 * sizeof(long long));
      B2RL_CUDA(cudaFuncSetAttribute(k_update_small, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)US_SMEM_BYTES));
      attr_set = true;
    }
    // chunks are applied in stream order, so last-writer-wins also holds across chunks
    for (int64_t off = 0; off < n; off += US_THREADS) {
      const int m = (int)((n - off < US_THREADS) ? (n - off) : US_THREADS);
      const bool last = off + US_THREADS >= n;
      k_update_small<<<1, US_THREADS, US_SMEM_BYTES, st>>>(t, idx_dev ? idx_dev + off : nullptr,
                                                           (ring_start + off) % h->capacity, h->capacity,
                                                           vals_dev ? vals_dev + off : nullptr, const_val, m, ks,
                                                           (publish_size_too && last) ? h->n_valid_dev : nullptr,
                                                           (float)h->size, probe);
      count_launch();
      if (probe) {      // debug: B2RL_TREE_PROBE=1 prints thread 0's cycle stamps of every small update
        long long hp[16];
        cudaStreamSynchronize(st);
        cudaMemcpy(hp, probe, sizeof(hp), cudaMemcpyDeviceToHost);
        fprintf(stderr, "[k_update_small n=%d ks=%d idx=%d] preload+sync %lld | winner+leaf %lld | sync %lld |", m, ks,
                idx_dev != nullptr, hp[1] - hp[0], hp[2] - hp[1], hp[3] - hp[2]);
        for (int k = 1; k <= ks; ++k) fprintf(stderr, " L%d %lld |", k, hp[3 + k] - hp[2 + k]);
        fprintf(stderr, " smem levels %lld | total %lld cycles\n", hp[12] - hp[3 + ks], hp[12] - hp[0]);
      }
    }
    B2RL_CHECK_LAUNCH();
    return B2RL_OK;
  }
  // Large batch: leaves first, then the levels bottom-up.  A level with no more nodes than the batch has
  // entries is recomputed for ALL of its nodes (cheaper and contention-free: thousands of entries would
  // otherwise recompute the same few nodes); everything from the first <= 256-node level upwards is one
  // single-CTA launch (ncu: a 4096-node level in one CTA cost 30 of the 35 us).
  const unsigned g = grid_for(n, UPD_THREADS);
  int launches = 0;
  if (idx_dev) {
    k_update_tag<<<g, UPD_THREADS, 0, st>>>(idx_dev, h->capacity, n, h->tag);
    k_update_write<<<g, UPD_THREADS, 0, st>>>(t, idx_dev, h->capacity, vals_dev, const_val, n, h->tag);
    launches += 2;
  } else {
    k_update_range_write<<<g, UPD_THREADS, 0, st>>>(t, ring_start, h->capacity, vals_dev, const_val, n);
    launches += 1;
  }
  const int64_t a0 = ring_start, b0 = (ring_start + n <= h->capacity) ? ring_start + n : h->capacity;
  const int64_t a1 = 0, b1 = (ring_start + n <= h->capacity) ? 0 : ring_start + n - h->capacity;
  // per-level launches while a level is wider than one CTA handles at a stroke (256 nodes), then one launch for the rest
  int kt = 1;
  while (kt < t.G && (t.cap2 >> (4 * kt)) > 256) ++kt;
  for (int k = 1; k < kt; ++k) {
    const int64_t nk = t.cap2 >> (4 * k);
    if (idx_dev) {
      if (nk <= n) k_tree_level_all<<<grid_for(nk, 256), 256, 0, st>>>(t, k);
      else k_update_level<<<g, UPD_THREADS, 0, st>>>(t, k, idx_dev, h->capacity, n);
    } else {
      const int sh = 4 * k;
      int64_t cnt = ((b0 - 1) >> sh) - (a0 >> sh) + 1;
      if (b1 > a1) cnt += ((b1 - 1) >> sh) - (a1 >> sh) + 1;
      k_update_range_level<<<grid_for(cnt, UPD_THREADS), UPD_THREADS, 0, st>>>(t, k, a0, b0, a1, b1);
    }
    ++launches;
  }
  k_tree_top<<<1, 256, 0, st>>>(t, kt);
  count_launch(launches + 1);
  B2RL_CHECK_LAUNCH();
  return publish_size_too ? publish_size(h, st) : B2RL_OK;
}

extern "C" int b2rl_tree_build(b2rl_replay* h, const float* prios_dev, int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0 && n <= h->capacity, "n out of range");
  B2RL_REQUIRE(n == 0 || prios_dev != nullptr, "null priorities");
  B2RL_REQUIRE(h->dedup == nullptr, "a frame-deduplicated replay's slots are made live by b2rl_dedup_push");
  DeviceGuard g(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const TreeView& t = h->tree;
  const int fused_upto = (t.G - 1 < 3) ? t.G - 1 : 3;       // full 16-wide levels the leaf kernel resolves itself
  const unsigned ctas = (unsigned)((t.cap2 + BUILD_LEAVES - 1) / BUILD_LEAVES);
  // Small trees: the last CTA to finish builds the top levels itself (one launch).  Large trees: the per-CTA
  // fence + ticket costs more than the second launch it saves (2^23: 21.3 vs 15.5 us), so k_tree_top follows.
  static int ticket_max_ctas = -1;
  if (ticket_max_ctas < 0) {
    const char* e = getenv("B2RL_BUILD_TICKET_CTAS");
    ticket_max_ctas = e ? atoi(e) : 296;
  }
  unsigned int* ticket = ((int)ctas <= ticket_max_ctas) ? h->build_ticket : nullptr;
  if ((((uintptr_t)prios_dev) & 15u) == 0)
    k_build_leaves<true><<<ctas, BUILD_THREADS, 0, st>>>(t, prios_dev, n, fused_upto, ticket);
  else
    k_build_leaves<false><<<ctas, BUILD_THREADS, 0, st>>>(t, prios_dev, n, fused_upto, ticket);
  count_launch();
  if (ticket == nullptr) {
    k_tree_top<<<1, 256, 0, st>>>(t, fused_upto + 1);
    count_launch();
  }
  B2RL_CHECK_LAUNCH();
  h->size = n;
  h->head = (n == h->capacity) ? 0 : n;
  return publish_size(h, st);
}

static int sample_launch(b2rl_replay* h, const double* u01_dev, uint64_t seed, uint64_t rng_offset,
                         const uint64_t* rng_state, int64_t n, float beta, const float* max_w_dev,
                         int64_t* idx_out_dev, float* prob_out_dev, float* w_out_dev, const SmallFields& small,
                         cudaStream_t st) {
  k_tree_sample<<<grid_for(n, SAMPLE_THREADS), SAMPLE_THREADS, 0, st>>>(
      h->tree, u01_dev, seed, rng_offset, rng_state, n, h->n_valid_dev, beta, max_w_dev, idx_out_dev,
      prob_out_dev, w_out_dev, small);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_tree_sample(b2rl_replay* h, const double* u01_dev, uint64_t seed,
                                uint64_t rng_offset, int64_t n, float beta, const float* max_w_dev,
                                int64_t* idx_out_dev, float* prob_out_dev, float* w_out_dev,
                                void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0, "negative n");
  B2RL_REQUIRE(h->size > 0, "sampling from an empty replay");
  B2RL_REQUIRE(n == 0 || idx_out_dev != nullptr, "null idx_out");
  if (n == 0) return B2RL_OK;
  DeviceGuard g(h->device);
  SmallFields none{};
  return sample_launch(h, u01_dev, seed, rng_offset, nullptr, n, beta, max_w_dev, idx_out_dev, prob_out_dev,
                       w_out_dev, none, (cudaStream_t)stream);
}

extern "C" int b2rl_replay_seed(b2rl_replay* h, uint64_t seed, uint64_t counter, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->device);
  k_rng_seed<<<1, 1, 0, (cudaStream_t)stream>>>(h->rng_dev, seed, counter);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_tree_sample_stream(b2rl_replay* h, int64_t n, float beta, const float* max_w_dev,
                                       int64_t* idx_out_dev, float* prob_out_dev, float* w_out_dev,
                                       void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0, "negative n");
  B2RL_REQUIRE(h->size > 0, "sampling from an empty replay");
  B2RL_REQUIRE(n == 0 || idx_out_dev != nullptr, "null idx_out");
  if (n == 0) return B2RL_OK;
  DeviceGuard g(h->device);
  SmallFields none{};
  return sample_launch(h, nullptr, 0, 0, h->rng_dev, n, beta, max_w_dev, idx_out_dev, prob_out_dev, w_out_dev,
                       none, (cudaStream_t)stream);
}

extern "C" int b2rl_tree_sample_fetch(b2rl_replay* h, int64_t n, float beta, const float* max_w_dev,
                                      int64_t* idx_out_dev, float* prob_out_dev, float* w_out_dev,
                                      void* const* small_fields_out_dev, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0, "negative n");
  B2RL_REQUIRE(h->size > 0, "sampling from an empty replay");
  B2RL_REQUIRE(n == 0 || idx_out_dev != nullptr, "null idx_out");
  if (n == 0) return B2RL_OK;
  SmallFields small{};
  if (small_fields_out_dev) {
    for (int f = 0; f < h->n_fields; ++f) {
      if (small_fields_out_dev[f] == nullptr) continue;
      const int64_t b = h->field_bytes[f];
      B2RL_REQUIRE(b == 1 || b == 2 || b == 4 || b == 8,
                   "b2rl_tree_sample_fetch only fetches 1/2/4/8-byte fields (use b2rl_replay_gather for rows)");
      small.src[small.n] = h->field[f];
      small.dst[small.n] = (uint8_t*)small_fields_out_dev[f];
      small.bytes[small.n] = (int)b;
      small.n++;
    }
  }
  DeviceGuard g(h->device);
  return sample_launch(h, nullptr, 0, 0, h->rng_dev, n, beta, max_w_dev, idx_out_dev, prob_out_dev, w_out_dev,
                       small, (cudaStream_t)stream);
}

extern "C" int b2rl_philox_uniforms(uint64_t seed, uint64_t rng_offset, int64_t n, double* out_dev,
                                    void* stream) {
  B2RL_REQUIRE(n >= 0 && (n == 0 || out_dev), "bad arguments");
  if (n == 0) return B2RL_OK;
  k_philox_uniforms<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(seed, rng_offset, n, out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_tree_update(b2rl_replay* h, const int64_t* idx_dev, const float* vals_dev,
                                int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n >= 0, "negative n");
  B2RL_REQUIRE(n == 0 || (idx_dev && vals_dev), "null idx/vals");
  B2RL_REQUIRE(n < (int64_t)0xFFFFFFFFLL, "batch too large");
  DeviceGuard g(h->device);
  return b2rl_tree_update_impl(h, idx_dev, 0, vals_dev, 0.0f, n, (cudaStream_t)stream, false);
}

extern "C" int b2rl_tree_stats(b2rl_replay* h, float beta, double* stats_out_dev, float* max_w_out_dev,
                               void* stream) {
  B2RL_REQUIRE(h != nullptr && (stats_out_dev != nullptr || max_w_out_dev != nullptr), "null argument");
  DeviceGuard g(h->device);
  k_tree_stats<<<1, 1, 0, (cudaStream_t)stream>>>(h->tree, h->n_valid_dev, beta, stats_out_dev, max_w_out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_tree_leaves(b2rl_replay* h, int64_t start, int64_t n, float* out_dev, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(start >= 0 && n >= 0 && start + n <= h->capacity, "range out of bounds");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(out_dev != nullptr, "null out");
  DeviceGuard g(h->device);
  k_tree_leaves<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(h->tree, start, n, out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_tree_level(const b2rl_replay* h, int32_t k, int64_t* n_nodes, int32_t* levels, int32_t* top_bits,
                               double* sums_out_dev, float* mins_out_dev, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(n_nodes != nullptr, "null n_nodes");
  const TreeView& t = h->tree;
  B2RL_REQUIRE(k >= 0 && k <= t.G, "no such stored level (0..G)");
  if (levels) *levels = t.G;
  if (top_bits) *top_bits = t.top_bits;
  if (k == 0) { *n_nodes = t.cap2; return B2RL_OK; }
  const int64_t nk = (k == t.G) ? 1 : (t.cap2 >> (4 * k));
  *n_nodes = nk;
  DeviceGuard g(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (sums_out_dev)
    B2RL_CUDA(cudaMemcpyAsync(sums_out_dev, t.sum + t.off[k], sizeof(double) * (size_t)nk, cudaMemcpyDeviceToDevice, st));
  if (mins_out_dev)
    B2RL_CUDA(cudaMemcpyAsync(mins_out_dev, t.minv + t.off[k], sizeof(float) * (size_t)nk, cudaMemcpyDeviceToDevice, st));
  return B2RL_OK;
}
