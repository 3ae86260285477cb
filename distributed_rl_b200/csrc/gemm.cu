// fp32-accurate dense layers on the tensor cores: C[M][N] (+)= A[M][K] * B[N][K]^T with 3xTF32.
//
// The dense heads of the Q-network (3136 -> 512, twice; cfg/ape_x.json:52-71) run as cuBLAS fp32
// SIMT GEMMs at PyTorch's default precision and are the largest share of the learner step (DESIGN.md §6b).
// TF32 alone (10-bit mantissa) is not what the reference computes, so every fp32 operand is split
//      x = hi + lo,   hi = rn_tf32(x),  lo = x - hi   (exact in fp32)
// and the product is formed as  hi*hi + hi*lo + lo*hi  with wgmma (tf32 inputs, fp32 accumulation in
// registers); the dropped lo*lo term is 2^-22 relative.  SURVEY.md §8f rank 2 ("TF32x3 policy").
//
//   k_split_pack   fp32 matrix (optionally transposed) -> {hi, lo} operand images in exactly the
//                  64B-swizzled, K-major tile layout the MMA reads, so the GEMM's loader is a
//                  plain cp.async.bulk per tile (no tensor map, no SM-side staging)
//   k_gemm_tf32x3  one CTA per (m-tile 128, n-tile 256, K-split): a TMA loader warp that keeps four 16-float
//                  half-chunk stages in flight, and two consumer warpgroups (64 rows each, 6 x wgmma m64n256k8
//                  per half-chunk) that store the tile (or, when K is split, this split's partial tile) straight
//                  from their accumulators
//   k_splitk_reduce sums the K-split partials in split order: the result is deterministic (no atomics).
//                  b2rl_gemm_tf32x3_partials leaves the partials in memory instead, for a consumer that sums them
//                  in the same order while it reads its input (k_dueling_forward, k_unflatten_relu_mask)
#include "common.cuh"
#include "hopper.cuh"
#include "operand_image.cuh"

namespace b2rl {
namespace gemm {

using namespace sm90;

constexpr int TM = 128, TN = 256;                   // tile rows of A / of B
constexpr int KC = image::KC, KH = image::KH;        // floats per K chunk (the split unit) / per staged half-chunk
constexpr int A_TILE = TM * KH * 4, B_TILE = TN * KH * 4;   // bytes of one {term, k_half} tile: 8 KiB / 16 KiB
constexpr int STAGE = 2 * A_TILE + 2 * B_TILE;       // hi+lo of both operands: 48 KiB
constexpr int STAGES = 4;                            // the loader runs up to three half-chunks ahead of the MMAs
// wgmma groups (one per half-chunk) a warpgroup leaves in flight before it releases a stage: the stage of
// half-chunk i - WG_DEPTH is refilled once half-chunk i's MMAs are issued
constexpr int WG_DEPTH = 1;
static_assert(WG_DEPTH >= 0 && WG_DEPTH < STAGES, "a released stage must not be one the MMAs still read");
constexpr int CONSUMERS = 256;                       // warpgroups 0-1: MMA + epilogue
constexpr int THREADS = CONSUMERS + 32;              // warp 8: TMA loader

// ---- operand packing ---------------------------------------------------------
// Image layout: operand_image.cuh.  One CTA per (32 operand rows, one K chunk); thread = (row r = tid / 8, 16-byte unit = tid % 8), so
// the source row segment is one contiguous 128 B per 8 threads, and each image row half one contiguous 64 B per 4.
// TRANSPOSE: the operand's rows are the source's columns; the 32x32 block goes through SMEM so that
// the source is still read along its contiguous dimension.
template <bool TRANSPOSE>
__global__ void __launch_bounds__(256)
k_split_pack(const float* __restrict__ src, int src_rows, int src_cols, int64_t src_ld, int tile_rows,
             float* __restrict__ out, int rows_pad, int k_chunks, int row_off, int kc_off) {
  // (row, kc) below are local to this piece; the image position is (row_off + row, kc_off + kc)
  const int kc = blockIdx.y, row0 = blockIdx.x * 32;
  const int r = threadIdx.x >> 3, unit = threadIdx.x & 7;
  const int row = row0 + r;
  float v[4];
  if (TRANSPOSE) {
    __shared__ float tile[32][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = kc * KC + w * 4 + j, c = row0 + lane;            // source row k, source column c
      tile[w * 4 + j][lane] = (k < src_rows && c < src_cols) ? src[(int64_t)k * src_ld + c] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = tile[unit * 4 + e][r];
  } else {
    const int k = kc * KC + unit * 4;
    const float* p = src + (int64_t)row * src_ld + k;
    if (row < src_rows && k + 3 < src_cols && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
      const float4 q = *reinterpret_cast<const float4*>(p);
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = (row < src_rows && k + e < src_cols) ? p[e] : 0.0f;
    }
  }
  const int irow = row_off + row, ikc = kc_off + kc;
  if (irow >= rows_pad) return;
  image::store_unit(out, image::offset(irow, ikc * KC + unit * 4, tile_rows, rows_pad), image::term_stride(k_chunks, rows_pad),
                    v);
}

// ---- activation-side packs that fold act_3 (ReLU) + nn.Flatten into the heads' operand images ----------------
// The conv stack's output is NHWC in memory: y[b][hw][c].  The reference flattens the logical NCHW tensor
// (baseline/baseNetwork.py:204-209), so the heads' weights index features as f = c*HW + hw.  Instead of a ReLU
// kernel plus a permuting copy per pass, these kernels read y coalesced, transpose through shared memory and write
// the operand images in f order directly (the weights' packs stay as they are).
//   k_pack_act_nhwc<false>: A-role image of x = relu(y) viewed [B][K = C*HW]          (forward)
//   k_pack_act_nhwc<true> : B-role image of x^T [K rows][contraction B]               (weight gradient)
//   k_unflatten_relu_mask : dL/dy[b][hw][c] = gx[b][c*HW + hw] * (y[b][hw][c] > 0)    (input gradient)
constexpr int ACT_PAD = 1;      // shared-memory row padding: kills the bank conflicts of the transposed reads

template <bool TRANSPOSE>
__global__ void __launch_bounds__(256)
k_pack_act_nhwc(const float* __restrict__ y, int B, int HW, int C, int relu, float* __restrict__ out,
                int rows_pad, int k_chunks) {
  extern __shared__ float s_act[];
  const int K = C * HW;
  if (!TRANSPOSE) {
    // one CTA per image row b (rows >= B are zero padding): s[hw][c], row stride C + 1
    const int b = blockIdx.x;
    const int ld = C + ACT_PAD;
    const uint32_t magic_c = (uint32_t)((0x100000000ull + C - 1) / C);      // i / C == (i * magic) >> 32 for i < 2^24
    const uint32_t magic_hw = (uint32_t)((0x100000000ull + HW - 1) / HW);
    if (b < B) {
      const float* src = y + (int64_t)b * K;
      for (int i = threadIdx.x; i < K; i += 256) {
        float v = src[i];
        if (relu) v = fmaxf(v, 0.0f);
        const int hw = (int)__umulhi((uint32_t)i, magic_c);
        s_act[hw * ld + (i - hw * C)] = v;
      }
    }
    __syncthreads();
    const int64_t ts = image::term_stride(k_chunks, rows_pad);
    for (int w = threadIdx.x; w < k_chunks * 8; w += 256) {
      const int kc = w >> 3, unit = w & 7;
      const int f0 = kc * KC + unit * 4;
      int c = (int)__umulhi((uint32_t)f0, magic_hw), hw = f0 - c * HW;      // f = c*HW + hw, walked incrementally
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        v[e] = (b < B && f0 + e < K) ? s_act[hw * ld + c] : 0.0f;
        if (++hw == HW) { hw = 0; ++c; }
      }
      image::store_unit(out, image::offset(b, f0, TM, rows_pad), ts, v);
    }
  } else {
    // one CTA per (chunk of 32 b's, hw): s[b][c], row stride C + 1; image rows f = c*HW + hw, contraction = b
    const int kc = blockIdx.x, hw = blockIdx.y;
    const int ld = C + ACT_PAD;
    for (int i = threadIdx.x; i < 32 * C; i += 256) {
      const int bb = i / C, c = i - bb * C, b = kc * KC + bb;
      float v = (b < B) ? y[((int64_t)b * HW + hw) * C + c] : 0.0f;
      if (relu) v = fmaxf(v, 0.0f);
      s_act[bb * ld + c] = v;
    }
    __syncthreads();
    const int64_t ts = image::term_stride(k_chunks, rows_pad);
    for (int w = threadIdx.x; w < C * 8; w += 256) {
      const int c = w >> 3, unit = w & 7;
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = s_act[(unit * 4 + e) * ld + c];
      image::store_unit(out, image::offset(c * HW + hw, kc * KC + unit * 4, TN, rows_pad), ts, v);
    }
  }
}

// zero rows [K, rows_pad) of the x^T image (the padding of the last row tile)
__global__ void __launch_bounds__(256)
k_pack_zero_rows(float* __restrict__ out, int row0, int rows_pad, int k_chunks, int tile_rows) {
  const int64_t ts = image::term_stride(k_chunks, rows_pad);
  const int n_rows = rows_pad - row0;
  const int64_t total = (int64_t)n_rows * k_chunks * 8;
  const float zero[4] = {0.f, 0.f, 0.f, 0.f};
  for (int64_t w = (int64_t)blockIdx.x * 256 + threadIdx.x; w < total; w += (int64_t)gridDim.x * 256) {
    const int unit = (int)(w & 7);
    const int64_t q = w >> 3;
    const int kc = (int)(q / n_rows), f = row0 + (int)(q - (int64_t)kc * n_rows);
    image::store_unit(out, image::offset(f, kc * KC + unit * 4, tile_rows, rows_pad), ts, zero);
  }
}

// gx: `splits` K-split partials of dL/dx, `split_stride` floats apart, summed here in split order (the same sum
// k_splitk_reduce forms)
__global__ void __launch_bounds__(256)
k_unflatten_relu_mask(const float* __restrict__ gx, int64_t gx_ld, int splits, int64_t split_stride,
                      const float* __restrict__ y, int HW, int C, float* __restrict__ out) {
  extern __shared__ float s_act[];          // gx row in f order: s[c*HW + hw]
  const int b = blockIdx.x, K = C * HW;
  const float* gr = gx + (int64_t)b * gx_ld;
  for (int i = threadIdx.x; i < K; i += 256) {
    float v = gr[i];
    for (int z = 1; z < splits; ++z) v += gr[z * split_stride + i];
    s_act[i] = v;
  }
  __syncthreads();
  const float* yr = y + (int64_t)b * K;
  float* o = out + (int64_t)b * K;
  for (int i = threadIdx.x; i < K; i += 256) {      // i = hw*C + c (coalesced reads of y, writes of out)
    const int hw = i / C, c = i - hw * C;
    o[i] = (yr[i] > 0.0f) ? s_act[c * HW + hw] : 0.0f;
  }
}

struct Params {
  const float* a;        // packed A image (tile_rows = 128)
  const float* b;        // packed B image (tile_rows = 256)
  float* c;              // splits == 1: C [M][ldc] fp32 (stored); else the partials [split][M][ldc]
  int64_t M, N, ldc;     // logical sizes (rows beyond M / columns beyond N are dropped)
  int64_t m_tiles, n_tiles, k_chunks;
  int32_t splits;        // K splits (gridDim.z)
};

__global__ void __launch_bounds__(THREADS, 1)
k_gemm_tf32x3(const __grid_constant__ Params P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (sptr(smem_raw) & 1023u)) & 1023u);
  __shared__ __align__(8) uint64_t full[STAGES], empty[STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t mt = blockIdx.x, nt = blockIdx.y;
  // K range of this split, in 32-float chunks; staged and multiplied as 2 (k1 - k0) half-chunks from 2 k0 on
  const int64_t per = (P.k_chunks + P.splits - 1) / P.splits;
  const int64_t k0 = (int64_t)blockIdx.z * per;
  const int64_t k1 = (k0 + per < P.k_chunks) ? k0 + per : P.k_chunks;
  const int64_t nk = 2 * (k1 - k0);   // > 0: the host never launches an empty trailing split (gemm_splits)

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMERS); }
    mbar_init_fence();
  }
  __syncthreads();
  if (nk <= 0) return;

  if (warp == CONSUMERS / 32) {
    // ------------------------------ TMA loader ------------------------------
    if (lane == 0) {
      const int64_t a_term = P.k_chunks * P.m_tiles * (TM * KC);   // floats between the hi and lo images
      const int64_t b_term = P.k_chunks * P.n_tiles * (TN * KC);
      for (int64_t i = 0; i < nk; ++i) {
        const int s = (int)(i % STAGES);
        mbar_wait(&empty[s], ((i / STAGES) & 1) ^ 1);
        const int64_t kh = 2 * k0 + i;
        const float* a_hi = P.a + (kh * P.m_tiles + mt) * (TM * KH);
        const float* b_hi = P.b + (kh * P.n_tiles + nt) * (TN * KH);
        uint8_t* st = smem + (size_t)s * STAGE;
        mbar_expect_tx(&full[s], STAGE);
        bulk_g2s(st, a_hi, A_TILE, &full[s]);
        bulk_g2s(st + A_TILE, a_hi + a_term, A_TILE, &full[s]);
        bulk_g2s(st + 2 * A_TILE, b_hi, B_TILE, &full[s]);
        bulk_g2s(st + 2 * A_TILE + B_TILE, b_hi + b_term, B_TILE, &full[s]);
      }
    }
    return;
  }

  // ------------------------- consumers: wgmma + epilogue -------------------------
  const int wg = warp >> 2;                            // rows [64 wg, 64 wg + 64) of the tile
  float acc[128];
#pragma unroll 1       // unrolled, the remainder path makes ptxas serialize the wgmmas (C7520)
  for (int64_t i = 0; i < nk; ++i) {
    const int s = (int)(i % STAGES);
    mbar_wait(&full[s], (i / STAGES) & 1);
    const uint32_t base = sptr(smem + (size_t)s * STAGE);
    const uint32_t a_hi = base + wg * (64 * KH * 4), a_lo = a_hi + A_TILE, b_hi = base + 2 * A_TILE, b_lo = b_hi + B_TILE;
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < KH / 8; ++ks) {
      const uint32_t o = ks * 32;
      mma_tf32_n256(acc, make_desc_sw64(a_lo + o), make_desc_sw64(b_hi + o), (i | ks) ? 1u : 0u);   // small terms first
      mma_tf32_n256(acc, make_desc_sw64(a_hi + o), make_desc_sw64(b_lo + o), 1u);
      mma_tf32_n256(acc, make_desc_sw64(a_hi + o), make_desc_sw64(b_hi + o), 1u);
    }
    wg_commit();
    wg_wait<WG_DEPTH>();                               // the MMAs of half-chunk i - WG_DEPTH are done: refill its stage
    wg_fence_regs(acc);
    if (i >= WG_DEPTH) mbar_arrive(&empty[(i - WG_DEPTH) % STAGES]);
  }
  wg_wait<0>();
  wg_fence_regs(acc);
  // fragment (see hopper.cuh): rows r0 and r0 + 8, columns 8j + 2(lane % 4) + {0, 1}
  const int64_t r0 = mt * TM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  float* cz = P.c + (int64_t)blockIdx.z * P.M * P.ldc;
#pragma unroll
  for (int j = 0; j < TN / 8; ++j) {
    const int64_t n = nt * TN + 8 * j + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t m = r0 + 8 * h;
      if (m >= P.M || n >= P.N) continue;
      float* dst = cz + m * P.ldc + n;
      if (n + 1 < P.N) *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      else dst[0] = acc[4 * j + 2 * h];
    }
  }
}

// C[i] = sum over splits (in split order: deterministic) of partial[z][i]; one thread per 4 columns
__global__ void __launch_bounds__(256)
k_splitk_reduce(const float* __restrict__ partial, int splits, int64_t M, int64_t N, int64_t ldc, float* __restrict__ c) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t per_row = ldc >> 2;
  if (q >= M * per_row) return;
  const int64_t m = q / per_row, n = (q - m * per_row) << 2;
  if (n >= N) return;
  const int64_t off = m * ldc + n, stride = M * ldc;
  if (n + 3 < N) {
    float4 a = *reinterpret_cast<const float4*>(partial + off);
    for (int z = 1; z < splits; ++z) {
      const float4 b = *reinterpret_cast<const float4*>(partial + z * stride + off);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    *reinterpret_cast<float4*>(c + off) = a;
  } else {
    for (int e = 0; n + e < N; ++e) {
      float a = partial[off + e];
      for (int z = 1; z < splits; ++z) a += partial[z * stride + off + e];
      c[off + e] = a;
    }
  }
}

}  // namespace gemm
}  // namespace b2rl

using namespace b2rl;

extern "C" int64_t b2rl_gemm_packed_floats(int64_t rows, int64_t k, int32_t b_role) {
  const int64_t tr = b_role ? gemm::TN : gemm::TM;
  const int64_t rows_pad = (rows + tr - 1) / tr * tr, kc = (k + gemm::KC - 1) / gemm::KC;
  return 2 * rows_pad * kc * gemm::KC;
}

// One piece of an operand: the piece's rows go to image rows [row_offset, ...), its contraction index to
// [k_offset, ...) of an operand with total_rows x total_k.  Pieces tile the operand (vertically stacked weight
// matrices, or their transposes side by side); the piece that ends the operand also writes the zero padding.
extern "C" int b2rl_gemm_split_pack_into(const float* src_dev, int64_t src_rows, int64_t src_cols, int64_t src_ld,
                                         int32_t transpose, int32_t b_role, float* out_dev, int64_t total_rows,
                                         int64_t total_k, int64_t row_offset, int64_t k_offset, void* stream) {
  B2RL_REQUIRE(src_dev && out_dev, "null argument");
  B2RL_REQUIRE(src_rows >= 1 && src_cols >= 1 && src_ld >= src_cols, "bad shape");
  B2RL_REQUIRE(((uintptr_t)out_dev % 16) == 0, "packed operand must be 16-byte aligned");
  const int64_t rows = transpose ? src_cols : src_rows, k = transpose ? src_rows : src_cols;
  B2RL_REQUIRE(row_offset >= 0 && k_offset >= 0 && row_offset + rows <= total_rows && k_offset + k <= total_k,
               "piece outside the operand");
  B2RL_REQUIRE(row_offset % 32 == 0 && k_offset % gemm::KC == 0, "piece offsets must be multiples of 32");
  B2RL_REQUIRE((rows % 32 == 0 || row_offset + rows == total_rows) && (k % gemm::KC == 0 || k_offset + k == total_k),
               "an inner piece must be a multiple of 32 rows / 32 contraction elements");
  const int tr = b_role ? gemm::TN : gemm::TM;
  const int64_t rows_pad = (total_rows + tr - 1) / tr * tr, kc_total = (total_k + gemm::KC - 1) / gemm::KC;
  B2RL_REQUIRE(rows_pad < (1 << 30) && kc_total <= 65535, "operand too large");
  const int64_t rows_cover = (row_offset + rows == total_rows) ? rows_pad - row_offset : rows;
  const int64_t kc_cover = (k + gemm::KC - 1) / gemm::KC;
  dim3 grid((unsigned)(rows_cover / 32), (unsigned)kc_cover);
  if (transpose)
    gemm::k_split_pack<true><<<grid, 256, 0, (cudaStream_t)stream>>>(src_dev, (int)src_rows, (int)src_cols, src_ld, tr,
                                                                     out_dev, (int)rows_pad, (int)kc_total,
                                                                     (int)row_offset, (int)(k_offset / gemm::KC));
  else
    gemm::k_split_pack<false><<<grid, 256, 0, (cudaStream_t)stream>>>(src_dev, (int)src_rows, (int)src_cols, src_ld, tr,
                                                                      out_dev, (int)rows_pad, (int)kc_total,
                                                                      (int)row_offset, (int)(k_offset / gemm::KC));
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_gemm_split_pack(const float* src_dev, int64_t src_rows, int64_t src_cols, int64_t src_ld,
                                    int32_t transpose, int32_t b_role, float* out_dev, void* stream) {
  const int64_t rows = transpose ? src_cols : src_rows, k = transpose ? src_rows : src_cols;
  return b2rl_gemm_split_pack_into(src_dev, src_rows, src_cols, src_ld, transpose, b_role, out_dev, rows, k, 0, 0, stream);
}

// K chunks one split accumulates at most.  The tensor cores' fp32 accumulation does not round to nearest, so its
// error grows with the length of the chain (12 wgmma steps per chunk).  Measured on an H100 SXM (132 SMs, 700 W):
// IMPALA's 2592 -> 256 layer erred 11x more than cuBLAS fp32 on the same inputs with 81 chunks in one split (forward)
// and 107 per split (weight gradient, K = 20 480); with at most 32 chunks (3 splits of 27, 20 of 32), 4.0x and 3.4x.
// On 132 SMs the Ape-X and R2D2 heads split into at most 25 chunks, so 32 leaves their splits, and the rounding of
// their results, as they were.  Shorter caps cut the error further but add splits there: 8 slowed the Ape-X step by
// 7 % (0.85 -> 0.91 ms).
constexpr int64_t MAX_CHUNKS_PER_SPLIT = 32;

static int64_t gemm_splits(int64_t M, int64_t N, int64_t K, int sms) {
  const int64_t tiles = ((M + gemm::TM - 1) / gemm::TM) * ((N + gemm::TN - 1) / gemm::TN);
  const int64_t kc = (K + gemm::KC - 1) / gemm::KC;
  int64_t splits = sms / (tiles > 0 ? tiles : 1);      // cover the SMs about once (a function of the shape only)
  if (splits < 1) splits = 1;
  if (splits > kc) splits = kc;
  if (splits * MAX_CHUNKS_PER_SPLIT < kc) splits = (kc + MAX_CHUNKS_PER_SPLIT - 1) / MAX_CHUNKS_PER_SPLIT;
  const int64_t per = (kc + splits - 1) / splits;
  return (kc + per - 1) / per;                          // no empty trailing split
}

static int gemm_sms(int* out) {
  int dev = 0;
  B2RL_CUDA(cudaGetDevice(&dev));
  B2RL_CUDA(sm_count(dev, out));
  return B2RL_OK;
}

extern "C" int64_t b2rl_gemm_workspace_floats(int64_t M, int64_t N, int64_t K, int64_t ldc) {
  int sms = 0;
  if (gemm_sms(&sms) != B2RL_OK) return -1;
  const int64_t splits = gemm_splits(M, N, K, sms);
  return splits > 1 ? splits * M * ldc : 0;
}

// k_gemm_tf32x3 alone: C (splits == 1) or the K-split partials [split][M][ldc] stored at `out`
static int gemm_launch(const float* a_packed_dev, const float* b_packed_dev, float* out, int64_t M, int64_t N,
                       int64_t K, int64_t ldc, int64_t splits, cudaStream_t st) {
  int dev = 0;
  B2RL_CUDA(cudaGetDevice(&dev));
  const size_t smem_bytes = (size_t)gemm::STAGES * gemm::STAGE + 1024;
  B2RL_CUDA(set_max_dynamic_smem<gemm::k_gemm_tf32x3>(dev, smem_bytes));
  gemm::Params P{};
  P.a = a_packed_dev; P.b = b_packed_dev;
  P.c = out;
  P.M = M; P.N = N; P.ldc = ldc;
  P.m_tiles = (M + gemm::TM - 1) / gemm::TM;
  P.n_tiles = (N + gemm::TN - 1) / gemm::TN;
  P.k_chunks = (K + gemm::KC - 1) / gemm::KC;
  P.splits = (int32_t)splits;
  dim3 grid((unsigned)P.m_tiles, (unsigned)P.n_tiles, (unsigned)splits);
  gemm::k_gemm_tf32x3<<<grid, gemm::THREADS, smem_bytes, st>>>(P);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_gemm_tf32x3_partials(const float* a_packed_dev, const float* b_packed_dev, float* partials_dev,
                                         int64_t M, int64_t N, int64_t K, int64_t ldc, void* stream) {
  B2RL_REQUIRE(a_packed_dev && b_packed_dev && partials_dev, "null argument");
  B2RL_REQUIRE(M >= 1 && N >= 1 && K >= 1 && ldc >= N, "bad shape");
  B2RL_REQUIRE(((uintptr_t)partials_dev % 16) == 0 && (ldc % 4) == 0,
               "partials must be 16-byte aligned with ldc % 4 == 0");
  int sms = 0;
  if (int rc = gemm_sms(&sms)) return rc;
  return gemm_launch(a_packed_dev, b_packed_dev, partials_dev, M, N, K, ldc, gemm_splits(M, N, K, sms),
                     (cudaStream_t)stream);
}

extern "C" int b2rl_gemm_tf32x3(const float* a_packed_dev, const float* b_packed_dev, float* c_dev, int64_t M,
                                int64_t N, int64_t K, int64_t ldc, float* workspace_dev, void* stream) {
  B2RL_REQUIRE(a_packed_dev && b_packed_dev && c_dev, "null argument");
  B2RL_REQUIRE(M >= 1 && N >= 1 && K >= 1 && ldc >= N, "bad shape");
  B2RL_REQUIRE(((uintptr_t)c_dev % 16) == 0 && (ldc % 4) == 0, "C must be 16-byte aligned with ldc % 4 == 0");
  int sms = 0;
  if (int rc = gemm_sms(&sms)) return rc;
  const int64_t splits = gemm_splits(M, N, K, sms);
  B2RL_REQUIRE(splits == 1 || (workspace_dev && ((uintptr_t)workspace_dev % 16) == 0),
               "this shape splits K: pass b2rl_gemm_workspace_floats() floats of 16-byte aligned workspace");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = gemm_launch(a_packed_dev, b_packed_dev, splits > 1 ? workspace_dev : c_dev, M, N, K, ldc, splits, st))
    return rc;
  if (splits > 1) {
    const int64_t quads = M * (ldc >> 2);
    gemm::k_splitk_reduce<<<(unsigned)((quads + 255) / 256), 256, 0, st>>>(workspace_dev, (int)splits, M, N, ldc, c_dev);
    count_launch();
    B2RL_CHECK_LAUNCH();
  }
  return B2RL_OK;
}


// flatten_NCHW(relu(y)) packed straight from the conv stack's NHWC output: act_3 + nn.Flatten of cfg/ape_x.json:37-51
// (baseline/baseNetwork.py:204-209) folded into the heads' operand packing.  transpose = 0: A-role image of
// x [B][C*HW] (forward); transpose = 1: B-role image of x^T (weight gradient of the heads).
extern "C" int b2rl_gemm_pack_act_nhwc(const float* y_dev, int64_t B, int64_t HW, int64_t C, int32_t relu, int32_t transpose,
                                       float* out_dev, void* stream) {
  B2RL_REQUIRE(y_dev && out_dev, "null argument");
  B2RL_REQUIRE(B >= 1 && HW >= 1 && C >= 1 && C * HW < (1 << 24) && B < (1 << 24), "bad shape");
  B2RL_REQUIRE(((uintptr_t)out_dev % 16) == 0, "packed operand must be 16-byte aligned");
  const int64_t K = C * HW;
  cudaStream_t st = (cudaStream_t)stream;
  if (!transpose) {
    const int64_t rows_pad = (B + gemm::TM - 1) / gemm::TM * gemm::TM, kc = (K + gemm::KC - 1) / gemm::KC;
    const size_t smem = (size_t)HW * (C + gemm::ACT_PAD) * sizeof(float);
    B2RL_REQUIRE(smem <= 48 * 1024, "activation row too large for the staging tile");
    gemm::k_pack_act_nhwc<false><<<(unsigned)rows_pad, 256, smem, st>>>(y_dev, (int)B, (int)HW, (int)C, relu, out_dev,
                                                                       (int)rows_pad, (int)kc);
    count_launch();
  } else {
    const int64_t rows_pad = (K + gemm::TN - 1) / gemm::TN * gemm::TN, kc = (B + gemm::KC - 1) / gemm::KC;
    const size_t smem = (size_t)32 * (C + gemm::ACT_PAD) * sizeof(float);
    B2RL_REQUIRE(smem <= 48 * 1024 && HW <= 65535, "activation tile too large");
    gemm::k_pack_act_nhwc<true><<<dim3((unsigned)kc, (unsigned)HW), 256, smem, st>>>(y_dev, (int)B, (int)HW, (int)C, relu,
                                                                                    out_dev, (int)rows_pad, (int)kc);
    count_launch();
    if (rows_pad > K) {
      gemm::k_pack_zero_rows<<<64, 256, 0, st>>>(out_dev, (int)K, (int)rows_pad, (int)kc, gemm::TN);
      count_launch();
    }
  }
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

// The backward counterpart: dL/dy (NHWC, [B][HW][C]) = dL/dx (NCHW-flatten order, [B][gx_ld]) permuted back and
// masked by the ReLU (y > 0) — nn.Flatten's and act_3's backward in one launch.
extern "C" int b2rl_unflatten_relu_mask(const float* gx_dev, int64_t gx_ld, int32_t splits, int64_t split_stride,
                                        const float* y_dev, int64_t B, int64_t HW, int64_t C, float* out_dev,
                                        void* stream) {
  B2RL_REQUIRE(gx_dev && y_dev && out_dev, "null argument");
  B2RL_REQUIRE(B >= 1 && HW >= 1 && C >= 1 && gx_ld >= C * HW, "bad shape");
  B2RL_REQUIRE(splits >= 1 && (splits == 1 || split_stride >= B * gx_ld), "bad split-K partials");
  const size_t smem = (size_t)C * HW * sizeof(float);
  B2RL_REQUIRE(smem <= 48 * 1024, "activation row too large for the staging tile");
  gemm::k_unflatten_relu_mask<<<(unsigned)B, 256, smem, (cudaStream_t)stream>>>(gx_dev, gx_ld, splits, split_stride,
                                                                              y_dev, (int)HW, (int)C, out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}
