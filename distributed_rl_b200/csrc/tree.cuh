// Device-side pieces of the sum-tree that more than one kernel uses: the 16-wide group loads, the radix-16
// descent of proportional sampling, the fetch of a sampled slot's scalar fields and the IS weight.
// k_tree_sample (tree.cu) and k_serve_fill (serve.cu) both draw through tree_draw / is_weight and fetch through
// fetch_small, so a served minibatch is bit-identical to b2rl_tree_sample_fetch from the same RNG state; its frame
// rows go through copy_rows (bulk_rows.cuh), as b2rl_replay_gather's.
#pragma once
#include "common.cuh"

#include <math.h>

namespace b2rl {

// Children of node `node` of stored level k (k >= 1) live on stored level k-1 at
// [node << bits, (node << bits) + 2^bits), bits = 4 below the top group.  Missing
// children of a narrower top group are 0 / +inf: x + 0 == x, so the pairwise sum
// is still the binary tree's value.
template <bool CG>
__device__ __forceinline__ float4 ld4f(const float* p) {
  return CG ? __ldcg(reinterpret_cast<const float4*>(p)) : *reinterpret_cast<const float4*>(p);
}
template <bool CG>
__device__ __forceinline__ double2 ld2d(const double* p) {
  return CG ? __ldcg(reinterpret_cast<const double2*>(p)) : *reinterpret_cast<const double2*>(p);
}

template <bool CG>
__device__ __forceinline__ void load_child_sums(const TreeView& t, int k, int64_t node, double c[16]) {
  const int bits = (k == t.G) ? t.top_bits : 4;
  if (k == 1) {
    const float* p = t.leaf + (node << bits);
    if (bits == 4) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v = ld4f<CG>(p + 4 * q);
        c[4 * q] = (double)v.x; c[4 * q + 1] = (double)v.y; c[4 * q + 2] = (double)v.z; c[4 * q + 3] = (double)v.w;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) c[i] = (i < (1 << bits)) ? (double)(CG ? __ldcg(p + i) : p[i]) : 0.0;
    }
  } else {
    const double* p = t.sum + t.off[k - 1] + (node << bits);
    if (bits == 4) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const double2 v = ld2d<CG>(p + 2 * q);
        c[2 * q] = v.x; c[2 * q + 1] = v.y;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) c[i] = (i < (1 << bits)) ? (CG ? __ldcg(p + i) : p[i]) : 0.0;
    }
  }
}

// Four binary descent steps inside one 16-wide group (Node._find :53-62 applied to the
// three recomputed levels and the stored children).  Returns the child index, updates pos,
// and leaves the selected child's sum in `picked`.
__device__ __forceinline__ int descend16(const double c_in[16], double& pos, double& picked) {
  double c[16], s1[8], s2[4], s3[2];
#pragma unroll
  for (int i = 0; i < 16; ++i) c[i] = c_in[i];
#pragma unroll
  for (int i = 0; i < 8; ++i) s1[i] = c[2 * i] + c[2 * i + 1];
#pragma unroll
  for (int i = 0; i < 4; ++i) s2[i] = s1[2 * i] + s1[2 * i + 1];
  s3[0] = s2[0] + s2[1];
  s3[1] = s2[2] + s2[3];
  // The `right == 0` guard only matters when pos rounds up to the subtree total (the reference
  // dereferences None there); it also steers a narrower top group into its zero-padded left part.
  const bool r1 = !((pos < s3[0]) || (s3[1] == 0.0));
  if (r1) pos = __dsub_rn(pos, s3[0]);
  const double a2 = r1 ? s2[2] : s2[0], b2 = r1 ? s2[3] : s2[1];
#pragma unroll
  for (int i = 0; i < 4; ++i) s1[i] = r1 ? s1[4 + i] : s1[i];
#pragma unroll
  for (int i = 0; i < 8; ++i) c[i] = r1 ? c[8 + i] : c[i];
  const bool r2 = !((pos < a2) || (b2 == 0.0));
  if (r2) pos = __dsub_rn(pos, a2);
  const double a1 = r2 ? s1[2] : s1[0], b1 = r2 ? s1[3] : s1[1];
#pragma unroll
  for (int i = 0; i < 4; ++i) c[i] = r2 ? c[4 + i] : c[i];
  const bool r3 = !((pos < a1) || (b1 == 0.0));
  if (r3) pos = __dsub_rn(pos, a1);
  const double a0 = r3 ? c[2] : c[0], b0 = r3 ? c[3] : c[1];
  const bool r4 = !((pos < a0) || (b0 == 0.0));
  if (r4) pos = __dsub_rn(pos, a0);
  picked = r4 ? b0 : a0;
  return (r1 ? 8 : 0) | (r2 ? 4 : 0) | (r3 ? 2 : 0) | (r4 ? 1 : 0);
}

// One proportional draw for the uniform u (SumTree.prioritized_sample, baseline/sumtree.py:128-140): the slot id;
// `root` receives the tree total and `picked` the drawn leaf's priority (as fp64).
__device__ __forceinline__ int64_t tree_draw(const TreeView& t, double u, double& root, double& picked) {
  root = t.sum[t.off[t.G]];
  double pos = __dmul_rn(root, u);  // np.random.uniform(0, root) == root * random_sample()
  int64_t node = 0;
  picked = 0.0;
  for (int lvl = t.G; lvl >= 1; --lvl) {
    double c[16];
    load_child_sums<false>(t, lvl, node, c);     // 128 B (64 B on the leaf level): one dependent load per 4 levels
    const int bits = (lvl == t.G) ? t.top_bits : 4;
    const int ch = descend16(c, pos, picked);
    node = (node << bits) | (int64_t)(ch & ((1 << bits) - 1));
  }
  return node;
}

struct SmallFields {
  const uint8_t* src[B2RL_MAX_FIELDS];
  uint8_t* dst[B2RL_MAX_FIELDS];
  int bytes[B2RL_MAX_FIELDS];
  int n;
};

// Scalar fields of sampled slot j (a, r, done: 1/2/4/8-byte rows) -> row k of the outputs.
__device__ __forceinline__ void fetch_small(const SmallFields& small, int64_t j, int64_t k) {
  for (int f = 0; f < small.n; ++f) {
    const int b = small.bytes[f];
    const uint8_t* s = small.src[f] + j * b;
    uint8_t* d = small.dst[f] + k * b;
    if (b == 4) *reinterpret_cast<uint32_t*>(d) = *reinterpret_cast<const uint32_t*>(s);
    else if (b == 1) *d = *s;
    else if (b == 8) *reinterpret_cast<uint64_t*>(d) = *reinterpret_cast<const uint64_t*>(s);
    else *reinterpret_cast<uint16_t*>(d) = *reinterpret_cast<const uint16_t*>(s);
  }
}

// APE_X/ReplayMemory.py:65-67, baseline/PER.py:98,129-133 — fp32 op by op.  s32 = (float)root, prob = p / s32.
__device__ __forceinline__ float is_weight(const TreeView& t, float s32, float prob, const float* n_valid_dev,
                                           float beta, const float* max_w_ext) {
  const float n_valid = *n_valid_dev;   // current number of valid slots (stream-ordered, not a launch constant)
  const float w_un = powcr(__fdiv_rn(1.0f, __fmul_rn(n_valid, prob)), beta);
  float max_w;
  if (max_w_ext) {
    max_w = *max_w_ext;
  } else {
    const float min_prob = __fdiv_rn(t.minv[t.off[t.G]], s32);
    max_w = powcr(__fmul_rn(n_valid, min_prob), -beta);
  }
  return __fdiv_rn(w_un, max_w);
}

// Device-resident Philox stream {seed, counter, ticket}: every block reads {seed, counter}; the LAST block to have
// done so advances the counter by n (and re-arms the ticket), so no separate launch is needed.  Every block of the
// grid must call this.
__device__ __forceinline__ void rng_stream_take(uint64_t* rng_state, int64_t n, uint64_t& seed, uint64_t& offset) {
  seed = rng_state[0];
  offset = rng_state[1];
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned int* ticket = reinterpret_cast<unsigned int*>(rng_state + 2);
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
      rng_state[1] = offset + (uint64_t)n;
      *ticket = 0u;
    }
  }
}

}  // namespace b2rl
