// Fused gather + first convolution of the Q-network on the Hopper tensor cores (wgmma).
//
//   y[k, oy, ox, co] = relu?( (1/255) * sum_{c,ky,kx} W[co, c, ky, kx] * frame[idx[k]][c, 4oy+ky, 4ox+kx] )
//
// for the 8x8 / stride-4 / 4->32 channel, bias-free conv_1 of cfg/ape_x.json and
// cfg/r2d2.json (baseline/baseNetwork.py:165-172), evaluated for up to two networks
// (online + target) in ONE pass over the sampled uint8 frame stacks.  It replaces,
// for the consumer of the gather, the staging copy + fp32 conversion + cuDNN conv
// (APE_X/Learner.py:61-67,78,85,87): the sampled rows go HBM -> SMEM (TMA bulk copy)
// -> im2col in SMEM -> wgmma -> registers -> NHWC fp32 activations, and the uint8
// frames are never written back to HBM.
//
// Arithmetic (DESIGN.md §4.6): the pixels are exact uint8, so the MMA runs on u8 x s8 -> s32
// (exact).  fp32 weights are split per output channel into four signed 7-bit digits,
// W = s * (q0 + q1/2^7 + q2/2^14 + q3/2^21) (+- s*2^-22), which are four groups of C_OUT
// columns of the same MMA (N = 128 per network).  The epilogue recombines the exact integer
// sums in fp32, so the result equals an fp32 convolution to ~2 ulp — tighter than cuDNN's
// TF32 path the reference would run.
//
// Warp roles per CTA (persistent, one CTA per SM, 17 warps):
//   warps 0-7    two consumer warpgroups, 64 rows of every 128-row tile each: per network
//                8 x wgmma m64nNk32 (N = 4 * C_OUT), then recombine digits -> scale -> ReLU ->
//                NHWC stores straight from the accumulator fragment
//   warps 8-15   im2col producers: SMEM frame -> 128B-swizzled K-major A tile (uint8);
//                thread = (tile row, channel pair)
//   warp 16      TMA loader: weights once, then one 28 224-byte frame stack per item, from the frame source of
//                frames.cuh: base + row * row_stride (a stride of 7 056 reads the overlapping 4-frame windows of a
//                frame strip: channel c of row r is frame r + c), or four 7 056-byte frames of a frame pool named by
//                a plane table
//
// A coded frame pool (FrameKind::CodedPlanes, b2rl_dedup_attach_coded) keeps the rule that the sampled frames never
// pass through HBM: the im2col producers decode them (frame_codec.cuh) straight into the raw buffers.  The encodings
// are read from global memory (a few hundred bytes per frame, L1/L2-resident once the row tables are prepared), and
// the loader warp loads only the weights.  The producers decode one frame of the next stack after each tile of the
// current one, and the rest after its last tile, so the consumers' MMAs on the staged A tiles overlap the decoding;
// raw buffer s is then handed over by a named barrier of the producers instead of raw_full / raw_empty.
#include "common.cuh"
#include "frames.cuh"
#include "hopper.cuh"

namespace b2rl {
namespace conv1 {

using namespace sm90;

constexpr int C_IN = 4, HW = 84, KS = 8, STRIDE = 4, OHW = 20;
constexpr int C_OUT_MAX = 32;                      // output channels: 32 (Ape-X / R2D2) or 16 (IMPALA), a template parameter
constexpr int K_TOTAL = C_IN * KS * KS;            // 256
constexpr int POS = OHW * OHW;                     // 400 output positions per frame stack
constexpr int TILE_M = 128;
constexpr int TILES = (POS + TILE_M - 1) / TILE_M; // 4 (the last one has 16 valid rows)
constexpr int NSPLIT = 4;
constexpr int A_STAGES = 2;
constexpr int A_TILE_BYTES = TILE_M * K_TOTAL;     // 32 768: 2 K-chunks x 128 rows x 128 B
constexpr int A_CHUNK_BYTES = TILE_M * 128;        // 16 384
constexpr int RAW_STRIDE = 28288;                  // STACK_BYTES rounded up to 128
constexpr int CONSUMERS = 256, PRODUCERS = 256;
constexpr int THREADS = CONSUMERS + PRODUCERS + 32;

// Byte offset of element (row n, k) inside a K-major SW128 operand with `rows` rows:
// [chunk = k/128][n/8][n%8][16-byte unit ^ (n%8)][byte]
__host__ __device__ __forceinline__ int sw128_offset(int rows, int n, int k) {
  const int j = k >> 7, kk = k & 127;
  return j * rows * 128 + (n >> 3) * 1024 + (n & 7) * 128 + ((((kk >> 4) ^ (n & 7))) << 4) + (kk & 15);
}

// ---- weight packing: fp32 [32][256] -> 4 signed 7-bit digits per weight, per-channel scale ----
__device__ __forceinline__ void pack_channel(const float* __restrict__ w, int net, int n_nets, int c_out, int co,
                                             int8_t* __restrict__ bq, float* __restrict__ scale) {
  __shared__ float s_max[K_TOTAL / 32];
  const int k = threadIdx.x;
  const float v = w[co * K_TOTAL + k];
  float m = fabsf(v);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((k & 31) == 0) s_max[k >> 5] = m;
  __syncthreads();
  m = s_max[0];
  for (int i = 1; i < K_TOTAL / 32; ++i) m = fmaxf(m, s_max[i]);
  const float s = (m > 0.0f) ? m / 127.0f : 1.0f;
  if (k == 0) scale[net * c_out + co] = s / 255.0f;   // the /255 of the input normalisation is folded in
  double x = (double)v / (double)s;
  const int rows = n_nets * NSPLIT * c_out;
#pragma unroll
  for (int j = 0; j < NSPLIT; ++j) {
    double q = rint(x);
    q = fmin(fmax(q, -127.0), 127.0);
    bq[sw128_offset(rows, net * NSPLIT * c_out + j * c_out + co, k)] = (int8_t)q;
    x = (x - q) * 128.0;
  }
}

__global__ void __launch_bounds__(K_TOTAL)
k_conv1_pack(const float* __restrict__ w, int net, int n_nets, int c_out, int8_t* __restrict__ bq,
             float* __restrict__ scale) {
  pack_channel(w, net, n_nets, c_out, blockIdx.x, bq, scale);
}

// Several packs in ONE launch (blockIdx.y = job): the learner step packs the online weights for its one-network and
// its two-network launch and the target weights for the latter — three launches in front of conv_1 became one.
constexpr int MAX_PACK_JOBS = 4;
struct PackJobs {
  const float* w[MAX_PACK_JOBS];
  int8_t* bq[MAX_PACK_JOBS];
  float* scale[MAX_PACK_JOBS];
  int32_t net[MAX_PACK_JOBS], n_nets[MAX_PACK_JOBS];
};
__global__ void __launch_bounds__(K_TOTAL)
k_conv1_pack_jobs(const __grid_constant__ PackJobs J, int c_out) {
  const int j = blockIdx.y;
  pack_channel(J.w[j], J.net[j], J.n_nets[j], c_out, blockIdx.x, J.bq[j], J.scale[j]);
}

struct Params {
  FrameSource src;           // where row r is read from (frames.cuh)
  const int64_t* idx;        // sampled rows, or nullptr for rows 0..n-1
  int64_t n;                 // frame stacks to process
  const int8_t* bq;          // packed weights (n_nets * 128 rows, SW128 layout), n_nets*128*256 bytes
  const float* scale;        // [n_nets][32] = s_c / 255
  float* out;                // [n_nets][n][400][32] fp32 (NHWC)
  int relu;
};

template <int N> struct Acc;
template <> struct Acc<128> {
  int32_t d[64];
  __device__ __forceinline__ void mma(uint64_t a, uint64_t b, uint32_t acc) { mma_u8s8_n128(d, a, b, acc); }
};
template <> struct Acc<64> {
  int32_t d[32];
  __device__ __forceinline__ void mma(uint64_t a, uint64_t b, uint32_t acc) { mma_u8s8_n64(d, a, b, acc); }
};

template <int N_NETS, int C_OUT, FrameKind KIND>
__global__ void __launch_bounds__(THREADS, 1)
k_conv1_fused(const __grid_constant__ Params P) {
  constexpr int N_PER_NET = NSPLIT * C_OUT;            // MMA columns per network: 128 (64 for 16 channels)
  constexpr int N_TOTAL = N_NETS * N_PER_NET;          // rows of the packed weights: 64 .. 256
  constexpr int B_BYTES = N_TOTAL * K_TOTAL;           // 16 .. 64 KiB
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // SWIZZLE_128B atoms must be 1024-byte aligned in the shared window: align by hand (1 KiB slack reserved)
  uint8_t* smem = smem_raw + ((1024u - (sptr(smem_raw) & 1023u)) & 1023u);
  uint8_t* sB = smem;
  uint8_t* sA = smem + B_BYTES;
  uint8_t* sRaw = sA + A_STAGES * A_TILE_BYTES;
  FcRows* sRows = reinterpret_cast<FcRows*>(sRaw + 2 * RAW_STRIDE);   // CodedPlanes: the decoders' row tables
  __shared__ __align__(8) uint64_t b_full, raw_full[2], raw_empty[2], a_full[A_STAGES], a_empty[A_STAGES];
  __shared__ float s_scale[2 * C_OUT_MAX];
  if (threadIdx.x < N_NETS * C_OUT) s_scale[threadIdx.x] = P.scale[threadIdx.x] * (1.0f / 128.0f);   // exact

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(&b_full, 1);
    for (int i = 0; i < 2; ++i) { mbar_init(&raw_full[i], 1); mbar_init(&raw_empty[i], PRODUCERS); }
    for (int i = 0; i < A_STAGES; ++i) { mbar_init(&a_full[i], PRODUCERS); mbar_init(&a_empty[i], CONSUMERS); }
    mbar_init_fence();
  }
  __syncthreads();
  // Work is split by (frame stack, 128-row tile) unit, not by frame stack: 512 stacks over 132 CTAs would be
  // 4 vs 3.88 stacks (16 vs 15.5 tiles); a CTA takes a contiguous run of units and loads every stack it touches.
  const int64_t units = P.n * TILES;
  const int64_t u0 = units * blockIdx.x / gridDim.x, u1 = units * (blockIdx.x + 1) / gridDim.x;
  const int64_t k_first = u0 / TILES, k_end = (u1 + TILES - 1) / TILES;   // stacks [k_first, k_end)

  if (warp == (CONSUMERS + PRODUCERS) / 32) {
    // ------------------------------ TMA loader ------------------------------
    if (lane == 0) {
      const uint8_t* frames = frame_base<KIND>(P.src);
      mbar_expect_tx(&b_full, B_BYTES);
      constexpr int LOAD_CHUNK = (B_BYTES < 32768) ? B_BYTES : 32768;
      for (int off = 0; off < B_BYTES; off += LOAD_CHUNK) bulk_g2s(sB + off, P.bq + off, LOAD_CHUNK, &b_full);
      if constexpr (KIND != FrameKind::CodedPlanes) {
        int it = 0;
        for (int64_t k = k_first; k < k_end; ++k, ++it) {
          const int s = it & 1;
          mbar_wait(&raw_empty[s], ((it >> 1) & 1) ^ 1);
          int64_t row = P.idx ? P.idx[k] : k;
          row = row < 0 ? 0 : (row >= P.src.rows ? P.src.rows - 1 : row);
          load_row<KIND>(P.src, frames, row, sRaw + s * RAW_STRIDE, &raw_full[s]);
        }
      }
    }
  } else if (warp >= CONSUMERS / 32) {
    // --------------------------- im2col producers ---------------------------
    const int pt = threadIdx.x - CONSUMERS;      // 0..255
    const int r_local = pt & (TILE_M - 1);       // A-tile row
    const int chalf = pt >> 7;                   // this thread converts channels 2*chalf, 2*chalf+1 (one K chunk)
    // CodedPlanes: frame c of stack k -> raw buffer `raw`, decoded by the eight producer warps together
    const int pw = pt >> 5;
    auto decode = [&](int64_t k, int c, uint8_t* raw) {
      int64_t row = P.idx ? P.idx[k] : k;
      row = row < 0 ? 0 : (row >= P.src.rows ? P.src.rows - 1 : row);
      decode_frame<PRODUCERS / 32>(coded_frame(P.src, row, c), raw + c * PLANE_BYTES, sRows, c & 1, 1, pw, lane);
    };
    if constexpr (KIND == FrameKind::CodedPlanes) {
      if (k_first < k_end) {
#pragma unroll 1
        for (int c = 0; c < C_IN; ++c) decode(k_first, c, sRaw);
        named_sync(1, PRODUCERS);
      }
    }
    int at = 0, it = 0;
    for (int64_t k = k_first; k < k_end; ++k, ++it) {
      const int s = it & 1;
      if constexpr (KIND != FrameKind::CodedPlanes) mbar_wait(&raw_full[s], (it >> 1) & 1);
      const uint8_t* raw = sRaw + s * RAW_STRIDE;
      // CodedPlanes: buffer s ^ 1 was last read for stack k - 1, before the barrier that ended it
      uint8_t* raw_next = sRaw + (s ^ 1) * RAW_STRIDE;
      int c_next = k + 1 < k_end ? 0 : C_IN;     // frames of stack k + 1 decoded so far
      const int t_lo = (int)max((int64_t)0, u0 - k * TILES), t_hi = (int)min((int64_t)TILES, u1 - k * TILES);
      for (int t = t_lo; t < t_hi; ++t, ++at) {
        const int stage = at % A_STAGES;
        mbar_wait(&a_empty[stage], ((at / A_STAGES) & 1) ^ 1);
        const int p = t * TILE_M + r_local;
        if (p < POS) {
          const int oy = p / OHW, ox = p - oy * OHW;
          const uint8_t* src_row = raw + (STRIDE * oy) * HW + STRIDE * ox + (2 * chalf) * (HW * HW);
          uint8_t* dst_row = sA + stage * A_TILE_BYTES + chalf * A_CHUNK_BYTES + (r_local >> 3) * 1024 +
                             (r_local & 7) * 128;
          const int sw = r_local & 7;
#pragma unroll
          for (int cc = 0; cc < 2; ++cc) {
#pragma unroll
            for (int kp = 0; kp < 4; ++kp) {
              const uint32_t* s0 = reinterpret_cast<const uint32_t*>(src_row + cc * (HW * HW) + (2 * kp) * HW);
              const uint32_t* s1 = reinterpret_cast<const uint32_t*>(src_row + cc * (HW * HW) + (2 * kp + 1) * HW);
              uint4 v;
              v.x = s0[0]; v.y = s0[1]; v.z = s1[0]; v.w = s1[1];
              const int unit = cc * 4 + kp;
              *reinterpret_cast<uint4*>(dst_row + ((unit ^ sw) << 4)) = v;
            }
          }
        }
        fence_async_smem();            // generic-proxy writes -> visible to the tensor core (async proxy)
        mbar_arrive(&a_full[stage]);
        if constexpr (KIND == FrameKind::CodedPlanes)
          if (c_next < C_IN) decode(k + 1, c_next++, raw_next);
      }
      if constexpr (KIND == FrameKind::CodedPlanes) {
#pragma unroll 1
        for (; c_next < C_IN; ++c_next) decode(k + 1, c_next, raw_next);
        named_sync(1, PRODUCERS);      // stack k + 1 is in raw_next, and every producer is done reading raw
      } else {
        mbar_arrive(&raw_empty[s]);    // this thread is done reading the raw frame
      }
    }
  } else {
    // ------------------------- consumers: wgmma + epilogue -------------------------
    // Warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile; the networks run one after the other so that one
    // accumulator (N_PER_NET / 2 registers) is live at a time.  Thread fragment (hopper.cuh): rows r and r + 8,
    // columns 8j + 2(lane % 4) + {0, 1}; column d * C_OUT + co is digit d of channel co, so every thread holds
    // all four digits of its channels.
    const int wg = warp >> 2;
    const float relu_floor = P.relu ? 0.0f : -INFINITY;
    const int r_in = (warp & 3) * 16 + (lane >> 2);            // row inside the warpgroup's 64
    const int c_in = 2 * (lane & 3);
    mbar_wait(&b_full, 0);
    int at = 0;
    for (int64_t k = k_first; k < k_end; ++k) {
      const int t_lo = (int)max((int64_t)0, u0 - k * TILES), t_hi = (int)min((int64_t)TILES, u1 - k * TILES);
      for (int t = t_lo; t < t_hi; ++t, ++at) {
        const int stage = at % A_STAGES;
        mbar_wait(&a_full[stage], (at / A_STAGES) & 1);
        const int p0 = t * TILE_M + wg * 64;                    // first output position of this warpgroup's rows
        if (p0 >= POS) {                                        // the last tile's upper half holds no positions
          mbar_arrive(&a_empty[stage]);
          continue;
        }
        const uint32_t a_base = sptr(sA + stage * A_TILE_BYTES) + wg * (64 * 128), b_base = sptr(sB);
#pragma unroll 1
        for (int net = 0; net < N_NETS; ++net) {
          Acc<N_PER_NET> acc;
          wg_fence();
#pragma unroll
          for (int kk = 0; kk < K_TOTAL / 32; ++kk) {
            const uint64_t ad = make_desc(a_base + (kk >> 2) * A_CHUNK_BYTES + (kk & 3) * 32);
            const uint64_t bd = make_desc(b_base + (kk >> 2) * (N_TOTAL * 128) + net * (N_PER_NET * 128) + (kk & 3) * 32);
            acc.mma(ad, bd, kk > 0 ? 1u : 0u);
          }
          wg_commit();
          wg_wait<0>();
          wg_fence_regs(acc.d);
          if (net == N_NETS - 1) mbar_arrive(&a_empty[stage]);   // SMEM stage reusable: every MMA has read it
          const float* sc = s_scale + net * C_OUT;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int p = p0 + r_in + 8 * h;
            if (p >= POS) continue;
            float* orow = P.out + (((int64_t)net * P.n + k) * POS + p) * C_OUT;
#pragma unroll
            for (int jj = 0; jj < C_OUT / 8; ++jj) {
              float y[2];
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const int i = 4 * jj + 2 * h + c;                 // digit d sits C_OUT / 8 fragment columns further
                const int32_t q0 = acc.d[i], q1 = acc.d[i + C_OUT / 2], q2 = acc.d[i + C_OUT], q3 = acc.d[i + 3 * C_OUT / 2];
                // digits are recombined pairwise in exact integer arithmetic (|u| < 2^31):
                //   u = q0*2^7 + q1,  t = q2*2^7 + q3,   sum = (u + t*2^-14) * 2^-7
                // one fp32 rounding per conversion (2^-24 relative), then one FMA and the scale.
                const float fu = (float)(q0 * 128 + q1);
                const float ft = (float)(q2 * 128 + q3);
                const float v = __fmaf_rn(ft, 1.0f / 16384.0f, fu) * sc[8 * jj + c_in + c];   // sc holds s_c / (255 * 2^7)
                y[c] = fmaxf(v, relu_floor);
              }
              *reinterpret_cast<float2*>(orow + 8 * jj + c_in) = make_float2(y[0], y[1]);
            }
          }
        }
      }
    }
  }
}

template <int N_NETS, int C_OUT, FrameKind KIND>
constexpr size_t smem_bytes() {
  return (size_t)N_NETS * NSPLIT * C_OUT * K_TOTAL + (size_t)A_STAGES * A_TILE_BYTES + 2 * (size_t)RAW_STRIDE + 1024 +
         (KIND == FrameKind::CodedPlanes ? DECODE_TABLES * sizeof(FcRows) : 0);
}

}  // namespace conv1
}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_conv1_pack(const float* w_dev, int32_t net, int32_t n_nets, int32_t c_out, int8_t* bq_out_dev,
                               float* scale_out_dev, void* stream) {
  B2RL_REQUIRE(w_dev && bq_out_dev && scale_out_dev, "null argument");
  B2RL_REQUIRE(n_nets >= 1 && n_nets <= 2 && net >= 0 && net < n_nets, "n_nets must be 1 or 2");
  B2RL_REQUIRE(c_out == 16 || c_out == 32, "c_out must be 16 or 32");
  conv1::k_conv1_pack<<<c_out, conv1::K_TOTAL, 0, (cudaStream_t)stream>>>(w_dev, net, n_nets, c_out, bq_out_dev,
                                                                         scale_out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_conv1_pack_jobs(const float* const* w_dev, const int32_t* net, const int32_t* n_nets,
                                    int8_t* const* bq_out_dev, float* const* scale_out_dev, int32_t jobs,
                                    int32_t c_out, void* stream) {
  B2RL_REQUIRE(w_dev && net && n_nets && bq_out_dev && scale_out_dev, "null argument");
  B2RL_REQUIRE(jobs >= 1 && jobs <= conv1::MAX_PACK_JOBS, "1..4 pack jobs");
  B2RL_REQUIRE(c_out == 16 || c_out == 32, "c_out must be 16 or 32");
  conv1::PackJobs J{};
  for (int j = 0; j < jobs; ++j) {
    B2RL_REQUIRE(w_dev[j] && bq_out_dev[j] && scale_out_dev[j], "null pack job");
    B2RL_REQUIRE(n_nets[j] >= 1 && n_nets[j] <= 2 && net[j] >= 0 && net[j] < n_nets[j], "n_nets must be 1 or 2");
    J.w[j] = w_dev[j]; J.bq[j] = bq_out_dev[j]; J.scale[j] = scale_out_dev[j];
    J.net[j] = net[j]; J.n_nets[j] = n_nets[j];
  }
  conv1::k_conv1_pack_jobs<<<dim3(c_out, jobs), conv1::K_TOTAL, 0, (cudaStream_t)stream>>>(J, c_out);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

template <int N_NETS, int C_OUT, FrameKind KIND>
static cudaError_t conv1_launch(const conv1::Params& P, unsigned grid, cudaStream_t st) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess)
    e = set_max_dynamic_smem<conv1::k_conv1_fused<N_NETS, C_OUT, KIND>>(dev, conv1::smem_bytes<N_NETS, C_OUT, KIND>());
  if (e != cudaSuccess) return e;
  conv1::k_conv1_fused<N_NETS, C_OUT, KIND><<<grid, conv1::THREADS, conv1::smem_bytes<N_NETS, C_OUT, KIND>(), st>>>(P);
  return cudaSuccess;
}

extern "C" int b2rl_conv1_fused(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const int8_t* bq_dev,
                                const float* scale_dev, int32_t n_nets, int32_t c_out, float* out_dev, int32_t relu,
                                void* stream) {
  B2RL_REQUIRE(n >= 0, "negative n");
  conv1::Params P{};
  FrameKind kind;
  if (const int rc = check_frames(frames, P.src, kind)) return rc;
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(bq_dev && scale_dev && out_dev, "null argument");
  B2RL_REQUIRE(n_nets == 1 || n_nets == 2, "n_nets must be 1 or 2");
  B2RL_REQUIRE(c_out == 16 || c_out == 32, "c_out must be 16 or 32");
  B2RL_REQUIRE(((uintptr_t)bq_dev % 16 == 0) && ((uintptr_t)out_dev % 16 == 0),
               "packed weights and output must be 16-byte aligned");
  int dev = 0;
  B2RL_CUDA(cudaGetDevice(&dev));
  int sms = 0;
  B2RL_CUDA(sm_count(dev, &sms));
  P.idx = idx_dev, P.n = n, P.bq = bq_dev, P.scale = scale_dev, P.out = out_dev, P.relu = relu;
  const int64_t units = n * conv1::TILES;
  const unsigned grid = (unsigned)((units < sms) ? units : sms);
  cudaStream_t st = (cudaStream_t)stream;
  const cudaError_t e = with_frame_kind(kind, [&](auto K) {
    constexpr FrameKind KIND = decltype(K)::value;
    if (c_out == 32) return n_nets == 1 ? conv1_launch<1, 32, KIND>(P, grid, st) : conv1_launch<2, 32, KIND>(P, grid, st);
    return n_nets == 1 ? conv1_launch<1, 16, KIND>(P, grid, st) : conv1_launch<2, 16, KIND>(P, grid, st);
  });
  B2RL_CUDA(e);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}
