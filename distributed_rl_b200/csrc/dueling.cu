// Fused tail of the dueling Q-network: everything after the first dense layer of the two heads.
//
//   r      = relu(h)                                    h: [M][2H] pre-activations, advantage | value
//   adv_j  = sum_k r[k]     * Wa[j][k]                  cfg/ape_x.json:52-71 (MLP 3136-512-A and 3136-512-1),
//   val    = sum_k r[H + k] * Wv[k]                     Add / Mean / Substract nodes :72-88,
//   Q_j    = adv_j + val - mean_i(adv_i)                baseline/baseAgent.py:287-309 executes them in order
//
// In PyTorch this is 6 small kernels per forward pass (ReLU, a 512x6 SIMT GEMM, a GEMV, add, mean, sub)
// and about twice that in backward; three passes per learner step.  Here: one kernel forward (one warp per
// row, the (A+1) x H weights in SMEM), two kernels backward (row-wise dL/dh with the ReLU mask; column-slab
// reduction over the batch for dL/dWa, dL/dWv in a fixed order, so the result is deterministic).
#include "common.cuh"

namespace b2rl {
namespace dueling {

constexpr int MAX_A = 32, MAX_H = 1024, ROWS_PER_CTA = 4;

// [A][H] advantage weights then [H] value weights into SMEM (H % 32 == 0: float4 copies)
__device__ __forceinline__ void load_weights(float* s_w, const float* __restrict__ wa, const float* __restrict__ wv,
                                             int A, int H) {
  const int na = (A * H) >> 2, nv = H >> 2;
  for (int i = threadIdx.x; i < na; i += blockDim.x)
    reinterpret_cast<float4*>(s_w)[i] = reinterpret_cast<const float4*>(wa)[i];
  for (int i = threadIdx.x; i < nv; i += blockDim.x)
    reinterpret_cast<float4*>(s_w + A * H)[i] = reinterpret_cast<const float4*>(wv)[i];
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

constexpr int STAGE_UNROLL = 8;      // float4 loads in flight per thread while the CTA stages its rows of h

// q[m][j] ; one warp per row, lane owns columns lane, lane+32, ...; the A+1 dot products are accumulated as
// independent chains and reduced together so that the shuffle latencies overlap.
// h: `splits` K-split partials [split][M][2H] of the heads' first-layer GEMM, `split_stride` floats apart.  The CTA
// first stages its ROWS_PER_CTA rows in SMEM, summing the partials in split order (the sum k_splitk_reduce forms);
// every thread keeps STAGE_UNROLL independent float4 loads in flight per split, so the sum runs at memory speed
// although a warp owns a whole row afterwards.  h_out (may be null) receives the summed rows.
template <int A_MAX>
__global__ void __launch_bounds__(ROWS_PER_CTA * 32)
k_dueling_forward(const float* __restrict__ h, int splits, int64_t split_stride, int M, int H,
                  const float* __restrict__ wa, int A, const float* __restrict__ wv, float* __restrict__ q,
                  float* __restrict__ h_out) {
  extern __shared__ float s_w[];                       // [A + 1][H]: Wa rows, then Wv; then [ROWS_PER_CTA][2H] of h
  float* s_h = s_w + A * H + H;
  load_weights(s_w, wa, wv, A, H);
  {
    const int m0 = blockIdx.x * ROWS_PER_CTA;
    const int n4 = (min(ROWS_PER_CTA, M - m0) * 2 * H) >> 2;          // float4s of this CTA's rows (contiguous)
    const float4* src = reinterpret_cast<const float4*>(h + (int64_t)m0 * 2 * H);
    const int64_t z4 = split_stride >> 2;
    float4* dst = h_out ? reinterpret_cast<float4*>(h_out + (int64_t)m0 * 2 * H) : nullptr;
    for (int i0 = threadIdx.x; i0 < n4; i0 += ROWS_PER_CTA * 32 * STAGE_UNROLL) {
      float4 v[STAGE_UNROLL];
#pragma unroll
      for (int u = 0; u < STAGE_UNROLL; ++u) {
        const int i = i0 + u * ROWS_PER_CTA * 32;
        v[u] = (i < n4) ? src[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      for (int z = 1; z < splits; ++z) {
#pragma unroll
        for (int u = 0; u < STAGE_UNROLL; ++u) {
          const int i = i0 + u * ROWS_PER_CTA * 32;
          if (i < n4) {
            const float4 w = src[z * z4 + i];
            v[u].x += w.x; v[u].y += w.y; v[u].z += w.z; v[u].w += w.w;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < STAGE_UNROLL; ++u) {
        const int i = i0 + u * ROWS_PER_CTA * 32;
        if (i < n4) {
          reinterpret_cast<float4*>(s_h)[i] = v[u];
          if (dst) dst[i] = v[u];
        }
      }
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, m = blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5);
  if (m >= M) return;
  const float* hr = s_h + (threadIdx.x >> 5) * 2 * H;
  float s[A_MAX], val = 0.0f;
#pragma unroll
  for (int j = 0; j < A_MAX; ++j) s[j] = 0.0f;
  for (int k = lane; k < H; k += 32) {
    const float ra = fmaxf(hr[k], 0.0f), rv = fmaxf(hr[H + k], 0.0f);
    val = __fmaf_rn(rv, s_w[A * H + k], val);
#pragma unroll
    for (int j = 0; j < A_MAX; ++j)
      if (j < A) s[j] = __fmaf_rn(ra, s_w[j * H + k], s[j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    val = __fadd_rn(val, __shfl_xor_sync(0xffffffffu, val, o));
#pragma unroll
    for (int j = 0; j < A_MAX; ++j)
      if (j < A) s[j] = __fadd_rn(s[j], __shfl_xor_sync(0xffffffffu, s[j], o));
  }
  float mine = 0.0f, total = 0.0f;                     // lane j keeps adv_j
#pragma unroll
  for (int j = 0; j < A_MAX; ++j) {
    if (j < A) {
      total = __fadd_rn(total, s[j]);
      if (lane == j) mine = s[j];
    }
  }
  if (lane < A) q[(int64_t)m * A + lane] = __fsub_rn(__fadd_rn(mine, val), __fdiv_rn(total, (float)A));
}

// dL/dh[m][:] from dL/dQ[m][:]:  g_adv_j = gq_j - mean(gq),  g_val = sum(gq)
__global__ void __launch_bounds__(ROWS_PER_CTA * 32)
k_dueling_backward_h(const float* __restrict__ h, const float* __restrict__ gq, int M, int H,
                     const float* __restrict__ wa, int A, const float* __restrict__ wv, float* __restrict__ gh,
                     float* __restrict__ ga) {
  extern __shared__ float s_w[];
  load_weights(s_w, wa, wv, A, H);
  __syncthreads();
  const int lane = threadIdx.x & 31, m = blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5);
  if (m >= M) return;
  const float g = (lane < A) ? gq[(int64_t)m * A + lane] : 0.0f;
  const float gval = warp_sum(g);
  const float gadv = __fsub_rn(g, __fdiv_rn(gval, (float)A));     // lane j holds g_adv_j
  if (lane < A) ga[(int64_t)m * (A + 1) + lane] = gadv;            // row table for k_dueling_backward_w
  if (lane == 0) ga[(int64_t)m * (A + 1) + A] = gval;
  if (gh == nullptr) return;
  const float* hr = h + (int64_t)m * 2 * H;
  float* gr = gh + (int64_t)m * 2 * H;
  const int n = H >> 5;
  float ha[MAX_H / 32], hv[MAX_H / 32], s[MAX_H / 32];
#pragma unroll
  for (int i = 0; i < MAX_H / 32; ++i) {
    ha[i] = (i < n) ? hr[lane + 32 * i] : 0.0f;
    hv[i] = (i < n) ? hr[H + lane + 32 * i] : 0.0f;
    s[i] = 0.0f;
  }
  for (int j = 0; j < A; ++j) {
    const float gj = __shfl_sync(0xffffffffu, gadv, j);
#pragma unroll
    for (int i = 0; i < MAX_H / 32; ++i)
      if (i < n) s[i] = __fmaf_rn(gj, s_w[j * H + lane + 32 * i], s[i]);
  }
#pragma unroll
  for (int i = 0; i < MAX_H / 32; ++i) {
    if (i < n) {
      gr[lane + 32 * i] = ha[i] > 0.0f ? s[i] : 0.0f;
      gr[H + lane + 32 * i] = hv[i] > 0.0f ? __fmul_rn(gval, s_w[A * H + lane + 32 * i]) : 0.0f;
    }
  }
}

// dL/dWa[j][k] = sum_m g_adv_j[m] relu(h[m][k]),  dL/dWv[k] = sum_m g_val[m] relu(h[m][H+k]), from the
// per-row (g_adv, g_val) table `ga` written by k_dueling_backward_h.  One CTA per 8 columns of h (one 32-byte
// sector per row); lane = (column, row group), 32 rows per CTA iteration; sums are combined in a fixed order.
template <int A_MAX>
__global__ void __launch_bounds__(256)
k_dueling_backward_w(const float* __restrict__ h, const float* __restrict__ ga, int M, int H, int A,
                     float* __restrict__ gwa, float* __restrict__ gwv) {
  __shared__ float s_part[8][A_MAX][8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = lane & 7, rg = lane >> 3;
  const int col0 = (int)blockIdx.x * 8;
  const bool is_val = col0 >= H;
  const int col = col0 + c;
  float acc[A_MAX];
#pragma unroll
  for (int j = 0; j < A_MAX; ++j) acc[j] = 0.0f;
  for (int m0 = w * 4 + rg; m0 < M; m0 += 32 * 4) {      // 4 rows per thread in flight
    float r[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int m = m0 + 32 * b;
      r[b] = (m < M) ? fmaxf(h[(int64_t)m * 2 * H + col], 0.0f) : 0.0f;
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int m = m0 + 32 * b;
      if (m < M) {
        const float* g = ga + (int64_t)m * (A + 1);
        if (is_val) {
          acc[0] = __fmaf_rn(g[A], r[b], acc[0]);
        } else {
#pragma unroll
          for (int j = 0; j < A_MAX; ++j)
            if (j < A) acc[j] = __fmaf_rn(g[j], r[b], acc[j]);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < A_MAX; ++j) {
    float v = acc[j];
    v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 8));
    v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 16));
    if (rg == 0) s_part[w][j][c] = v;
  }
  __syncthreads();
  const int nj = is_val ? 1 : A;
  for (int t = threadIdx.x; t < nj * 8; t += blockDim.x) {
    const int j = t >> 3, cc = t & 7;
    float s = 0.0f;
#pragma unroll
    for (int ww = 0; ww < 8; ++ww) s = __fadd_rn(s, s_part[ww][j][cc]);
    if (is_val) gwv[col0 - H + cc] = s;
    else gwa[(int64_t)j * H + col0 + cc] = s;
  }
}

}  // namespace dueling
}  // namespace b2rl

using namespace b2rl;

static int dueling_check(const void* h, int64_t M, int64_t H, int64_t A) {
  B2RL_REQUIRE(h != nullptr, "null argument");
  B2RL_REQUIRE(M >= 1 && A >= 1 && A <= dueling::MAX_A, "actions must be 1..32");
  B2RL_REQUIRE(H >= 32 && H <= dueling::MAX_H && H % 32 == 0, "hidden width must be a multiple of 32, <= 1024");
  return B2RL_OK;
}

static cudaError_t dueling_smem(const void* fn, size_t bytes) {
  return bytes > 48 * 1024 ? cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes)
                           : cudaSuccess;
}

extern "C" int b2rl_dueling_forward(const float* h_dev, int32_t splits, int64_t split_stride, int64_t M, int64_t H,
                                    const float* wa_dev, int64_t A, const float* wv_dev, float* q_dev, float* h_out_dev,
                                    void* stream) {
  if (int rc = dueling_check(h_dev, M, H, A)) return rc;
  B2RL_REQUIRE(wa_dev && wv_dev && q_dev, "null argument");
  B2RL_REQUIRE(((uintptr_t)wa_dev % 16) == 0 && ((uintptr_t)wv_dev % 16) == 0, "weights must be 16-byte aligned");
  B2RL_REQUIRE(((uintptr_t)h_dev % 16) == 0 && ((uintptr_t)h_out_dev % 16) == 0, "h must be 16-byte aligned");
  B2RL_REQUIRE(splits >= 1 && (splits == 1 || (split_stride >= M * 2 * H && split_stride % 4 == 0)),
               "bad split-K partials");
  const size_t smem = (size_t)(A + 1 + 2 * dueling::ROWS_PER_CTA) * H * sizeof(float);
  const unsigned grid = (unsigned)((M + dueling::ROWS_PER_CTA - 1) / dueling::ROWS_PER_CTA);
  const unsigned block = dueling::ROWS_PER_CTA * 32;
  cudaStream_t st = (cudaStream_t)stream;
  if (A <= 8) {
    B2RL_CUDA(dueling_smem((const void*)dueling::k_dueling_forward<8>, smem));
    dueling::k_dueling_forward<8><<<grid, block, smem, st>>>(h_dev, splits, split_stride, (int)M, (int)H, wa_dev,
                                                                 (int)A, wv_dev, q_dev, h_out_dev);
  } else if (A <= 16) {
    B2RL_CUDA(dueling_smem((const void*)dueling::k_dueling_forward<16>, smem));
    dueling::k_dueling_forward<16><<<grid, block, smem, st>>>(h_dev, splits, split_stride, (int)M, (int)H, wa_dev,
                                                                 (int)A, wv_dev, q_dev, h_out_dev);
  } else {
    B2RL_CUDA(dueling_smem((const void*)dueling::k_dueling_forward<32>, smem));
    dueling::k_dueling_forward<32><<<grid, block, smem, st>>>(h_dev, splits, split_stride, (int)M, (int)H, wa_dev,
                                                                 (int)A, wv_dev, q_dev, h_out_dev);
  }
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_dueling_backward_w(const float* h_dev, const float* row_ws_dev, int64_t M, int64_t H, int64_t A,
                                       float* gwa_dev, float* gwv_dev, void* stream);

extern "C" int b2rl_dueling_backward(const float* h_dev, const float* gq_dev, int64_t M, int64_t H,
                                     const float* wa_dev, int64_t A, const float* wv_dev, float* gh_dev,
                                     float* gwa_dev, float* gwv_dev, float* row_ws_dev, void* stream) {
  if (int rc = dueling_check(h_dev, M, H, A)) return rc;
  B2RL_REQUIRE(gq_dev && wa_dev && wv_dev && row_ws_dev, "null argument");
  B2RL_REQUIRE(((uintptr_t)wa_dev % 16) == 0 && ((uintptr_t)wv_dev % 16) == 0, "weights must be 16-byte aligned");
  B2RL_REQUIRE((gwa_dev == nullptr) == (gwv_dev == nullptr), "both weight gradients or neither");
  cudaStream_t st = (cudaStream_t)stream;
  {
    const size_t smem = (size_t)(A + 1) * H * sizeof(float);
    B2RL_CUDA(dueling_smem((const void*)dueling::k_dueling_backward_h, smem));
    const unsigned grid = (unsigned)((M + dueling::ROWS_PER_CTA - 1) / dueling::ROWS_PER_CTA);
    dueling::k_dueling_backward_h<<<grid, dueling::ROWS_PER_CTA * 32, smem, st>>>(h_dev, gq_dev, (int)M, (int)H, wa_dev,
                                                                                 (int)A, wv_dev, gh_dev, row_ws_dev);
    count_launch();
    B2RL_CHECK_LAUNCH();
  }
  if (gwa_dev) return b2rl_dueling_backward_w(h_dev, row_ws_dev, M, H, A, gwa_dev, gwv_dev, stream);
  return B2RL_OK;
}

extern "C" int b2rl_dueling_backward_w(const float* h_dev, const float* row_ws_dev, int64_t M, int64_t H, int64_t A,
                                       float* gwa_dev, float* gwv_dev, void* stream) {
  if (int rc = dueling_check(h_dev, M, H, A)) return rc;
  B2RL_REQUIRE(row_ws_dev && gwa_dev && gwv_dev, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  {
    const unsigned grid = (unsigned)(2 * H / 8);
    if (A <= 8)
      dueling::k_dueling_backward_w<8><<<grid, 256, 0, st>>>(h_dev, row_ws_dev, (int)M, (int)H, (int)A, gwa_dev, gwv_dev);
    else if (A <= 16)
      dueling::k_dueling_backward_w<16><<<grid, 256, 0, st>>>(h_dev, row_ws_dev, (int)M, (int)H, (int)A, gwa_dev, gwv_dev);
    else
      dueling::k_dueling_backward_w<32><<<grid, 256, 0, st>>>(h_dev, row_ws_dev, (int)M, (int)H, (int)A, gwa_dev, gwv_dev);
    count_launch();
    B2RL_CHECK_LAUNCH();
  }
  return B2RL_OK;
}
