// Fused optimizer step for the learners' RMSprop (cfg/ape_x.json:27-35 centered, cfg/impala.json:19-23
// plain): ONE pass over (param, grad, square_avg, grad_avg) of every tensor that
//   * applies torch.optim.RMSprop's update (baseline/utils.py getOptim :124-130),
//   * zeroes the gradient (optim.zero_grad),
//   * accumulates per-tensor sum(g^2) for the reference's "norm" = sqrt(sum_i ||g_i||_2)
//     (APE_X/Learner.py:123-138, a per-tensor .norm() kernel + sync each in the reference).
// Replaces ~14 foreach / elementwise launches per step.  SURVEY.md §8f rank 2.
//
// A 2-D tensor may come with 3xTF32 operand images of itself (the dense heads' first-layer weights: the forward
// B operand and the W^T B operand of dL/dx, operand_image.cuh).  Its blocks then take 32x32 tiles and write both
// images from the updated values, so the images change exactly when the weights do and no GEMM has to repack them.
#include "common.cuh"
#include "operand_image.cuh"

namespace b2rl {

constexpr int OPT_MAX_TENSORS = 24;
constexpr int OPT_THREADS = 256;
constexpr int OPT_PER_THREAD = 4;
constexpr int64_t OPT_CHUNK = (int64_t)OPT_THREADS * OPT_PER_THREAD;

struct OptTable {
  float* p[OPT_MAX_TENSORS];
  float* g[OPT_MAX_TENSORS];
  float* sq[OPT_MAX_TENSORS];
  float* ga[OPT_MAX_TENSORS];
  int64_t numel[OPT_MAX_TENSORS];
  int32_t block_start[OPT_MAX_TENSORS + 1];   // first block of each tensor (a block never straddles tensors)
  // operand images (either may be null): fwd = B-role image of the weight stack [total_n rows][cols] (this tensor at
  // rows n_off..), wt = B-role image of its transpose [cols rows][total_n contraction] (at contraction n_off..)
  float* img_fwd[OPT_MAX_TENSORS];
  float* img_wt[OPT_MAX_TENSORS];
  int32_t cols[OPT_MAX_TENSORS];
  int32_t n_off[OPT_MAX_TENSORS];
  int32_t fwd_rows_pad[OPT_MAX_TENSORS], fwd_kc[OPT_MAX_TENSORS];
  int32_t wt_rows_pad[OPT_MAX_TENSORS], wt_kc[OPT_MAX_TENSORS];
  int32_t n_tensors;
};

// torch.optim.RMSprop's per-element update; returns the new parameter
__device__ __forceinline__ float rmsprop_elem(float p, float g, float& sq, float& ga, float lr, float alpha,
                                              float one_m_alpha, float eps, int centered) {
  sq = __fmaf_rn(one_m_alpha * g, g, sq * alpha);                   // square_avg.mul_(alpha).addcmul_(g, g, 1-alpha)
  float avg;
  if (centered) {
    ga = __fmaf_rn(one_m_alpha, g - ga, ga);                         // grad_avg.lerp_(g, 1-alpha)
    avg = __fsqrt_rn(__fmaf_rn(-ga, ga, sq));                        // addcmul(ga, ga, -1).sqrt_()
  } else {
    avg = __fsqrt_rn(sq);
  }
  return p - lr * (g / (avg + eps));                                 // addcdiv_(g, avg + eps, -lr)
}

__global__ void __launch_bounds__(OPT_THREADS)
k_rmsprop(const __grid_constant__ OptTable T, float lr, float alpha, float one_m_alpha, float eps, int centered,
          double* __restrict__ sumsq /*[n_tensors] or nullptr*/) {
  __shared__ double s_part[OPT_THREADS / 32];
  int t = 0;
  while (t + 1 < T.n_tensors && (int)blockIdx.x >= T.block_start[t + 1]) ++t;
  const int64_t base = (int64_t)(blockIdx.x - T.block_start[t]) * OPT_CHUNK;
  const int64_t n = T.numel[t];
  float* __restrict__ P = T.p[t];
  float* __restrict__ G = T.g[t];
  float* __restrict__ SQ = T.sq[t];
  float* __restrict__ GA = T.ga[t];
  double acc = 0.0;
  if (T.img_fwd[t] || T.img_wt[t]) {
    // a 32x32 tile of the [rows][cols] weight: thread = (row r, 4 columns of unit), one float4 of each array
    __shared__ float tile[32][33];
    const int tiles_k = T.cols[t] / image::KC;
    const int bt = (int)(blockIdx.x - T.block_start[t]), rt = bt / tiles_k, kc = bt - rt * tiles_k;
    const int r = threadIdx.x >> 3, unit = threadIdx.x & 7;
    const int64_t i0 = (int64_t)(rt * 32 + r) * T.cols[t] + kc * image::KC + unit * 4;
    float4 p4 = *reinterpret_cast<const float4*>(P + i0);
    const float4 g4 = *reinterpret_cast<const float4*>(G + i0);
    float4 sq4 = *reinterpret_cast<const float4*>(SQ + i0);
    float4 ga4 = centered ? *reinterpret_cast<const float4*>(GA + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
    float* pv = &p4.x;
    const float* gv = &g4.x;
    float* sqv = &sq4.x;
    float* gav = &ga4.x;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      pv[e] = rmsprop_elem(pv[e], gv[e], sqv[e], gav[e], lr, alpha, one_m_alpha, eps, centered);
      acc += (double)gv[e] * (double)gv[e];
    }
    *reinterpret_cast<float4*>(P + i0) = p4;
    *reinterpret_cast<float4*>(SQ + i0) = sq4;
    if (centered) *reinterpret_cast<float4*>(GA + i0) = ga4;
    *reinterpret_cast<float4*>(G + i0) = make_float4(0.f, 0.f, 0.f, 0.f);               // zero_grad
    if (T.img_fwd[t]) {          // image row = the weight's row n_off + rt*32 + r, contraction = its columns (k_split_pack<false>)
      const int rows_pad = T.fwd_rows_pad[t];
      image::store_unit(T.img_fwd[t], image::offset(T.n_off[t] + rt * 32 + r, kc * image::KC + unit * 4, 256, rows_pad),
                        image::term_stride(T.fwd_kc[t], rows_pad), pv);
    }
    if (T.img_wt[t]) {           // transposed through SMEM: image row = column kc*32 + r, contraction = stack rows (k_split_pack<true>)
#pragma unroll
      for (int e = 0; e < 4; ++e) tile[r][unit * 4 + e] = pv[e];
      __syncthreads();
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = tile[unit * 4 + e][r];
      const int rows_pad = T.wt_rows_pad[t];
      image::store_unit(T.img_wt[t], image::offset(kc * image::KC + r, T.n_off[t] + rt * 32 + unit * 4, 256, rows_pad),
                        image::term_stride(T.wt_kc[t], rows_pad), v);
    }
  } else {
#pragma unroll
    for (int u = 0; u < OPT_PER_THREAD; ++u) {
      const int64_t i = base + (int64_t)u * OPT_THREADS + threadIdx.x;
      if (i < n) {
        const float g = G[i];
        float sq = SQ[i], ga = centered ? GA[i] : 0.0f;
        P[i] = rmsprop_elem(P[i], g, sq, ga, lr, alpha, one_m_alpha, eps, centered);
        SQ[i] = sq;
        if (centered) GA[i] = ga;
        G[i] = 0.0f;                                                   // zero_grad
        acc += (double)g * (double)g;
      }
    }
  }
  if (sumsq) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int w = 0; w < OPT_THREADS / 32; ++w) s += s_part[w];
      atomicAdd(sumsq + t, s);     // diagnostic value only: fp64 accumulation, order matters at the 1e-16 level
    }
  }
}

__global__ void k_grad_norm_finish(double* __restrict__ sumsq, int n, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double s = 0.0;
  for (int i = 0; i < n; ++i) { s += sqrt(sumsq[i]); sumsq[i] = 0.0; }   // self-clean for the next step
  *out = (float)sqrt(s);                                      // "p_norm ** .5" of APE_X/Learner.py:130
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_rmsprop_step(float* const* params, float* const* grads, float* const* square_avg,
                                 float* const* grad_avg, const int64_t* numel, int32_t n_tensors, double lr,
                                 double alpha, double eps, int32_t centered, const int64_t* images,
                                 double* sumsq_scratch_dev, float* grad_norm_out_dev, void* stream) {
  B2RL_REQUIRE(n_tensors >= 1 && n_tensors <= OPT_MAX_TENSORS, "1..24 tensors");
  B2RL_REQUIRE(params && grads && square_avg && numel, "null argument");
  B2RL_REQUIRE(!centered || grad_avg, "centered RMSprop needs grad_avg");
  B2RL_REQUIRE(!grad_norm_out_dev || sumsq_scratch_dev,
               "the gradient norm needs a zero-initialised scratch of n_tensors doubles");
  OptTable T{};
  T.n_tensors = n_tensors;
  int64_t blocks = 0;
  for (int i = 0; i < n_tensors; ++i) {
    B2RL_REQUIRE(numel[i] >= 1 && params[i] && grads[i] && square_avg[i] && (!centered || grad_avg[i]),
                 "bad tensor entry");
    T.p[i] = params[i]; T.g[i] = grads[i]; T.sq[i] = square_avg[i]; T.ga[i] = centered ? grad_avg[i] : nullptr;
    T.numel[i] = numel[i];
    const int64_t* im = images ? images + 6 * i : nullptr;
    if (im && (im[0] || im[1])) {
      // {fwd image, W^T image, rows, cols, total_n, n_off}: the weight is rows x cols, row-major, in the stack of
      // total_n rows at n_off; both images cover the whole stack (b2rl_gemm_split_pack_into's total_rows / total_k)
      const int64_t rows = im[2], cols = im[3], total_n = im[4], n_off = im[5];
      B2RL_REQUIRE(rows >= 32 && cols >= 32 && rows % 32 == 0 && cols % 32 == 0 && rows * cols == numel[i] &&
                   n_off >= 0 && n_off % 32 == 0 && n_off + rows <= total_n && total_n < (1 << 30) &&
                   cols < (1 << 30), "image tensor: rows, cols and offsets must be multiples of 32 inside the stack");
      B2RL_REQUIRE(((uintptr_t)params[i] | (uintptr_t)grads[i] | (uintptr_t)square_avg[i] |
                    (uintptr_t)(centered ? grad_avg[i] : nullptr) | (uintptr_t)im[0] | (uintptr_t)im[1]) % 16 == 0,
                   "image tensor: 16-byte aligned arrays and images");
      T.img_fwd[i] = reinterpret_cast<float*>(im[0]);
      T.img_wt[i] = reinterpret_cast<float*>(im[1]);
      T.cols[i] = (int32_t)cols;
      T.n_off[i] = (int32_t)n_off;
      T.fwd_rows_pad[i] = (int32_t)((total_n + 255) / 256 * 256);
      T.fwd_kc[i] = (int32_t)(cols / image::KC);
      T.wt_rows_pad[i] = (int32_t)((cols + 255) / 256 * 256);
      T.wt_kc[i] = (int32_t)((total_n + image::KC - 1) / image::KC);
    }
    T.block_start[i] = (int32_t)blocks;
    blocks += (numel[i] + OPT_CHUNK - 1) / OPT_CHUNK;
  }
  T.block_start[n_tensors] = (int32_t)blocks;
  B2RL_REQUIRE(blocks < (1LL << 31), "too many elements");
  cudaStream_t st = (cudaStream_t)stream;
  // python-double hyper-parameters, cast once like torch's foreach kernels do (1 - alpha formed in double)
  k_rmsprop<<<(unsigned)blocks, OPT_THREADS, 0, st>>>(T, (float)lr, (float)alpha, (float)(1.0 - alpha), (float)eps,
                                                      centered, sumsq_scratch_dev);
  count_launch();
  if (grad_norm_out_dev) {
    k_grad_norm_finish<<<1, 32, 0, st>>>(sumsq_scratch_dev, n_tensors, grad_norm_out_dev);
    count_launch();
  }
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_rmsprop_norm_finish(double* sumsq_scratch_dev, int32_t n_tensors, float* grad_norm_out_dev,
                                        void* stream) {
  B2RL_REQUIRE(sumsq_scratch_dev && grad_norm_out_dev, "null argument");
  B2RL_REQUIRE(n_tensors >= 1 && n_tensors <= OPT_MAX_TENSORS, "1..24 tensors");
  k_grad_norm_finish<<<1, 32, 0, (cudaStream_t)stream>>>(sumsq_scratch_dev, n_tensors, grad_norm_out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}
