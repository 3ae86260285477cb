// The stem of the IMPALA residual network (agent.ResidualStack, Espeholt et al. 2018, Fig. 3): its first 3x3 / stride-1
// / pad-1, 4 -> 16 channel, bias-free conv and the 3x3 / stride-2 / pad-1 max-pool after it, fused with the gather of
// the sampled frame stacks, forward and weight gradient.
//
//   y[k, co, y, x]   = (1/255) * sum_{c,ky,kx} W[co, c, ky, kx] * frame[idx[k]][c, y+ky-1, x+kx-1]     (zero padding)
//   p[k, co, py, px] = max over the window rows 2py-1+i, cols 2px-1+j (i, j < 3) of y, padded positions skipped
//   a[k, co, py, px] = 3i + j of the FIRST maximum in (i, j) row-major order (torch's max_pool2d picks the same one)
//
// The frames go HBM -> SMEM (the TMA loaders of frames.cuh) -> a zero-bordered copy -> tensor cores, and are never
// staged as fp32; the 84x84x16 conv output never leaves the chip.  DESIGN.md §4.25.
//
// Arithmetic (conv_1's scheme, DESIGN.md §4.6): the pixels are exact uint8, so the MMA runs u8 x s8 -> s32 against four
// signed 7-bit digits of the weights (b2rl_conv1_pack's digit arithmetic), recombined in the epilogue as conv_1's are.
// The contraction K = 4 channels x 3 rows x 3 taps is laid out as 12 groups (c, ky) of four bytes, the fourth tap
// weighted by zero, so one 32-bit word of a group is four consecutive pixels of one frame row: K = 48 = one
// mma.m16n8k32 plus one mma.m16n8k16 per 16 positions and 8 output columns (N = 4 digits x 16 channels = 64).
//
// Forward: one frame stack per CTA at a time (persistent, two CTAs per SM, 8 warps).  The conv output is made in bands
// of six rows (504 positions = 32 m16 tiles, four per warp) into a ring of seven rows of SMEM, so the one-row halo the
// next band's pooled rows need (row 6b - 1) is kept from the band before; then the band's three pooled rows are
// max-pooled from the ring and written (pooled fp32 [n][16][42][42] NCHW, the layout the residual blocks' convs take,
// and the uint8 argmax [n][16][42][42]).  The loader prefetches the next stack while the CTA works on this one.
//
// Weight gradient: dW[co, e] = (1/255) sum_{k, y, x} gy[k, co, y, x] * X_e[k, y, x], with gy the conv output's gradient
// folded from the pooled gradient in the loader: position (y, x) of channel co sums, in (py, px) order, the pooled
// gradients of the (at most four) windows whose argmax chose it — deterministic, no atomics.  The stem's input is data,
// so no input gradient.  conv1_wgrad's scheme (DESIGN.md §4.10): gy as four balanced base-256 digits against a
// power-of-two scale pre-scanned per stack (s > 4 max|dL/dp| / 127 bounds every folded sum), u8 x s8 -> s32 MMAs over
// the stack's positions (M = 4 digits x 16 channels, N = 36 patch elements padded to 40), the exact digit sums of each
// stack recombined in int64 and added in fp64; per-warp sums added in warp order, per-CTA partials in CTA order in fp64.
#include "common.cuh"
#include "frames.cuh"
#include "hopper.cuh"

namespace b2rl {
namespace stem {

using namespace sm90;

constexpr int C_IN = 4, HW = 84, C_OUT = 16, PHW = 42;
constexpr int K_TAPS = 36;                         // (c, ky, kx)
constexpr int GROUPS = 12;                         // (c, ky): four bytes each, the fourth weighted by zero
constexpr int K_PAD = 4 * GROUPS;                  // 48
constexpr int NSPLIT = 4;                          // weight digits
constexpr int N_COLS = NSPLIT * C_OUT;             // 64: column d * 16 + co is digit d of channel co
constexpr int PAD_W = 88, PAD_H = 86;              // zero-bordered frame: pixel (r, x) at [r + 1][x + 1]
constexpr int PAD_PLANE = PAD_H * PAD_W;           // 7 568
constexpr int PAD_BYTES = C_IN * PAD_PLANE;        // 30 272
constexpr int RAW_BYTES = 28288;                   // STACK_BYTES rounded up to 128
constexpr int THREADS = 256, WARPS = THREADS / 32;
constexpr int POOLED = C_OUT * PHW * PHW;          // 28 224 pooled elements per stack
// forward
constexpr int BAND = 6;                            // conv rows made per band: three pooled rows
constexpr int BANDS = HW / BAND;                   // 14
constexpr int BAND_POS = BAND * HW;                // 504
constexpr int M_TILES = (BAND_POS + 15) / 16;      // 32
constexpr int RING = BAND + 1;                     // conv rows kept: the band and the row before it
constexpr int RING_BYTES = RING * C_OUT * HW * 4;  // 37 632
// weight gradient
constexpr int POS = HW * HW;                       // 7 056 conv positions per stack
constexpr int K_STEPS = (POS + 31) / 32;           // 221 (the last one half zeros)
constexpr int E_TILES = (K_TAPS + 7) / 8;          // 5 n8 tiles of patch elements
constexpr int WG_OUT = C_OUT * K_TAPS;             // 576 weight-gradient elements

__device__ __forceinline__ void mma_k32(int32_t (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_k16(int32_t (&d)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
               : "r"(a0), "r"(a1), "r"(b0));
}
__device__ __forceinline__ void mma_k32_s8u8(int32_t (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Four consecutive bytes of a zero-bordered frame row starting at byte `x` (any alignment).
__device__ __forceinline__ uint32_t pad_word(const uint8_t* row, int x) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(row + (x & ~3));
  return __funnelshift_r(w[0], w[1], 8 * (x & 3));
}

// Zero-bordered copy of the raw stack: padded row word w of frame row r is raw bytes 4w - 1 .. 4w + 2 (byte -1 and
// bytes 84.. are the zero border).  The border rows and columns are zeroed once by zero_pad.
__device__ __forceinline__ void fill_pad(const uint8_t* raw, uint8_t* pad) {
  constexpr int RAW_WORDS = HW / 4, PAD_WORDS = PAD_W / 4;    // 21, 22
  for (int i = threadIdx.x; i < C_IN * HW * PAD_WORDS; i += THREADS) {
    const int w = i % PAD_WORDS, cr = i / PAD_WORDS;           // cr = c * 84 + r
    const uint32_t* src = reinterpret_cast<const uint32_t*>(raw + cr * HW);
    const uint32_t lo = w > 0 ? src[w - 1] : 0u, hi = w < RAW_WORDS ? src[w] : 0u;
    const int c = cr / HW, r = cr - c * HW;
    reinterpret_cast<uint32_t*>(pad + c * PAD_PLANE + (r + 1) * PAD_W)[w] = __funnelshift_l(lo, hi, 8);
  }
}
__device__ __forceinline__ void zero_pad(uint8_t* pad) {
  for (int i = threadIdx.x; i < PAD_BYTES / 4; i += THREADS) reinterpret_cast<uint32_t*>(pad)[i] = 0u;
}

__device__ __forceinline__ int64_t clamp_row(const FrameSource& S, const int64_t* idx, int64_t k) {
  const int64_t row = idx ? idx[k] : k;
  return row < 0 ? 0 : (row >= S.rows ? S.rows - 1 : row);
}

// ---- weight packing: fp32 [16][4][3][3] -> four signed 7-bit digits per weight, per-channel scale ----
// The digits of b2rl_conv1_pack (conv1.cu pack_channel): s = max|W[co]| / 127, q_j = rint(x) clamped to +-127,
// x <- (x - q_j) * 128.  Layout bq[d * 16 + co][48]: byte 4 (3c + ky) + kx, byte 4g + 3 zero.
__global__ void __launch_bounds__(64) k_stem_pack(const float* __restrict__ w, int8_t* __restrict__ bq,
                                                  float* __restrict__ scale) {
  __shared__ float s_max[2];
  const int co = blockIdx.x, k = threadIdx.x;         // k < 36 a tap, 36..63 idle lanes of the second warp
  const float v = k < K_TAPS ? w[co * K_TAPS + k] : 0.0f;
  float m = fabsf(v);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((k & 31) == 0) s_max[k >> 5] = m;
  __syncthreads();
  m = fmaxf(s_max[0], s_max[1]);
  const float s = (m > 0.0f) ? m / 127.0f : 1.0f;
  if (k == 0) scale[co] = s / 255.0f;                  // the /255 of the input normalisation is folded in
  if (k >= K_TAPS) return;
  const int g = k / 3, kx = k - 3 * g;                 // k = 3 (3c + ky) + kx
  double x = (double)v / (double)s;
#pragma unroll
  for (int j = 0; j < NSPLIT; ++j) {
    double q = rint(x);
    q = fmin(fmax(q, -127.0), 127.0);
    int8_t* row = bq + (j * C_OUT + co) * K_PAD;
    row[4 * g + kx] = (int8_t)q;
    if (kx == 2) row[4 * g + 3] = 0;
    x = (x - q) * 128.0;
  }
}

struct FwdParams {
  FrameSource src;
  const int64_t* idx;        // sampled rows, or nullptr for rows 0..n-1
  int64_t n;
  const int8_t* bq;          // [64][48] packed digits
  const float* scale;        // [16] = s_c / 255
  float* pooled;             // [n][16][42][42]
  uint8_t* argmax;           // [n][16][42][42]
};

template <FrameKind KIND>
__global__ void __launch_bounds__(THREADS, 2)
k_stem_fused(const __grid_constant__ FwdParams P) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* sRaw = smem_raw;
  uint8_t* sPad = sRaw + RAW_BYTES;
  float* sRing = reinterpret_cast<float*>(sPad + PAD_BYTES);   // [7][16][84]: conv row r in slot (r + 1) % 7
  __shared__ __align__(8) uint64_t raw_full;
  __shared__ float s_scale[C_OUT];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gid = lane >> 2, tig = lane & 3;
  if (threadIdx.x < C_OUT) s_scale[threadIdx.x] = P.scale[threadIdx.x] * (1.0f / 128.0f);   // exact
  zero_pad(sPad);
  if (threadIdx.x == 0) {
    mbar_init(&raw_full, 1);
    mbar_init_fence();
  }
  __syncthreads();
  const uint8_t* frames = frame_base<KIND>(P.src);
  if (threadIdx.x == 0 && blockIdx.x < P.n)
    load_row<KIND>(P.src, frames, clamp_row(P.src, P.idx, blockIdx.x), sRaw, &raw_full);

  // weight fragments: n-tile j = columns 8j .. 8j + 7 (digit j / 2, channels 8 (j % 2) ..); b0 / b1 the k32 step's
  // groups tig and tig + 4, b2 the k16 step's group 8 + tig
  uint32_t bw[8][3];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t* row = reinterpret_cast<const uint32_t*>(P.bq + (8 * j + gid) * K_PAD);
    bw[j][0] = row[tig]; bw[j][1] = row[tig + 4]; bw[j][2] = row[tig + 8];
  }
  // this thread's A groups (c, ky): tig, tig + 4, tig + 8 -> byte offset of padded row ky of channel c
  int goff[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int g = tig + 4 * q;
    goff[q] = (g / 3) * PAD_PLANE + (g % 3) * PAD_W;
  }

  int it = 0;
  for (int64_t k = blockIdx.x; k < P.n; k += gridDim.x, ++it) {
    mbar_wait(&raw_full, it & 1);
    fill_pad(sRaw, sPad);
    fence_async_smem();            // every generic read of sRaw is ordered before the next bulk copy into it
    __syncthreads();
    if (threadIdx.x == 0 && k + gridDim.x < P.n)
      load_row<KIND>(P.src, frames, clamp_row(P.src, P.idx, k + gridDim.x), sRaw, &raw_full);
    float* pooled = P.pooled + k * POOLED;
    uint8_t* amax = P.argmax + k * POOLED;

#pragma unroll 1
    for (int b = 0; b < BANDS; ++b) {
      // ---- conv rows 6b .. 6b + 5 into the ring ----
#pragma unroll 1
      for (int t = warp; t < M_TILES; t += WARPS) {
        int yy[2], xx[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int p = min(t * 16 + gid + 8 * h, BAND_POS - 1);   // rows past the band compute a copy, not stored
          const int r = p / HW;
          yy[h] = BAND * b + r, xx[h] = p - r * HW;
        }
        uint32_t a[4], a4, a5;
        a[0] = pad_word(sPad + goff[0] + yy[0] * PAD_W, xx[0]);
        a[1] = pad_word(sPad + goff[0] + yy[1] * PAD_W, xx[1]);
        a[2] = pad_word(sPad + goff[1] + yy[0] * PAD_W, xx[0]);
        a[3] = pad_word(sPad + goff[1] + yy[1] * PAD_W, xx[1]);
        a4 = pad_word(sPad + goff[2] + yy[0] * PAD_W, xx[0]);
        a5 = pad_word(sPad + goff[2] + yy[1] * PAD_W, xx[1]);
        int32_t acc[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0;
          mma_k32(acc[j], a, bw[j][0], bw[j][1]);
          mma_k16(acc[j], a4, a5, bw[j][2]);
        }
        // fragment: acc[j][2h + c] = row gid + 8h, column 8j + 2 tig + c; digit d of channel co is column 16d + co,
        // so tile j = 2d + (co >= 8) and this thread holds all four digits of channels 2tig + c and 8 + 2tig + c
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (t * 16 + gid + 8 * h >= BAND_POS) continue;
          float* ring = sRing + ((yy[h] + 1) % RING) * (C_OUT * HW) + xx[h];
#pragma unroll
          for (int half = 0; half < 2; ++half) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int i = 2 * h + c;
              const int32_t q0 = acc[half][i], q1 = acc[2 + half][i], q2 = acc[4 + half][i], q3 = acc[6 + half][i];
              // conv1.cu's recombination: exact pairs, one fp32 rounding each, one FMA, the scale
              const float fu = (float)(q0 * 128 + q1);
              const float ft = (float)(q2 * 128 + q3);
              const int co = 8 * half + 2 * tig + c;
              ring[co * HW] = __fmaf_rn(ft, 1.0f / 16384.0f, fu) * s_scale[co];
            }
          }
        }
      }
      __syncthreads();
      // ---- pooled rows 3b .. 3b + 2 from conv rows 6b - 1 .. 6b + 5 ----
      for (int e = threadIdx.x; e < C_OUT * 3 * PHW; e += THREADS) {
        const int co = e / (3 * PHW), rem = e - co * (3 * PHW);
        const int py = 3 * b + rem / PHW, px = rem % PHW;
        float best = -INFINITY;
        int bi = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int y = 2 * py - 1 + i;
          if (y < 0) continue;                                     // padded row (y <= 83 always)
          const float* ring = sRing + ((y + 1) % RING) * (C_OUT * HW) + co * HW;
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            const int x = 2 * px - 1 + j;
            if (x < 0) continue;                                   // padded column (x <= 83 always)
            const float v = ring[x];
            if (v > best || v != v) { best = v; bi = 3 * i + j; }  // first maximum, as max_pool2d (NaN wins)
          }
        }
        const int o = co * (PHW * PHW) + py * PHW + px;
        pooled[o] = best;
        amax[o] = (uint8_t)bi;
      }
      __syncthreads();
    }
  }
}

// ---- the stem of two networks over the same rows (b2rl_stem_fused_pair) ----
// k_stem_fused's per-stack work as functions.  k_stem_fused keeps its own inline copy: routed through these, nvcc
// commutes a few address additions and its SASS would no longer be the one it has been measured and checked with.

// weight fragments of one pack: n-tile j = columns 8j .. 8j + 7 (digit j / 2, channels 8 (j % 2) ..); b0 / b1 the k32
// step's groups tig and tig + 4, b2 the k16 step's group 8 + tig
__device__ __forceinline__ void load_weight_frags(const int8_t* bq, int gid, int tig, uint32_t (&bw)[8][3]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t* row = reinterpret_cast<const uint32_t*>(bq + (8 * j + gid) * K_PAD);
    bw[j][0] = row[tig]; bw[j][1] = row[tig + 4]; bw[j][2] = row[tig + 8];
  }
}

// One stack against one pack: the 14 bands of conv rows from the zero-bordered image into the ring, each band's three
// pooled rows written to `pooled` (and, with ARGMAX, their argmax to `amax`).  Ends on a barrier: the ring is free.
template <bool ARGMAX>
__device__ __forceinline__ void conv_pool_stack(const uint8_t* sPad, float* sRing, const uint32_t (&bw)[8][3],
                                                const int (&goff)[3], const float* s_scale, float* pooled,
                                                uint8_t* amax, int warp, int gid, int tig) {
#pragma unroll 1
  for (int b = 0; b < BANDS; ++b) {
    // ---- conv rows 6b .. 6b + 5 into the ring ----
#pragma unroll 1
    for (int t = warp; t < M_TILES; t += WARPS) {
      int yy[2], xx[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int p = min(t * 16 + gid + 8 * h, BAND_POS - 1);   // rows past the band compute a copy, not stored
        const int r = p / HW;
        yy[h] = BAND * b + r, xx[h] = p - r * HW;
      }
      uint32_t a[4], a4, a5;
      a[0] = pad_word(sPad + goff[0] + yy[0] * PAD_W, xx[0]);
      a[1] = pad_word(sPad + goff[0] + yy[1] * PAD_W, xx[1]);
      a[2] = pad_word(sPad + goff[1] + yy[0] * PAD_W, xx[0]);
      a[3] = pad_word(sPad + goff[1] + yy[1] * PAD_W, xx[1]);
      a4 = pad_word(sPad + goff[2] + yy[0] * PAD_W, xx[0]);
      a5 = pad_word(sPad + goff[2] + yy[1] * PAD_W, xx[1]);
      int32_t acc[8][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0;
        mma_k32(acc[j], a, bw[j][0], bw[j][1]);
        mma_k16(acc[j], a4, a5, bw[j][2]);
      }
      // fragment: acc[j][2h + c] = row gid + 8h, column 8j + 2 tig + c; digit d of channel co is column 16d + co,
      // so tile j = 2d + (co >= 8) and this thread holds all four digits of channels 2tig + c and 8 + 2tig + c
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (t * 16 + gid + 8 * h >= BAND_POS) continue;
        float* ring = sRing + ((yy[h] + 1) % RING) * (C_OUT * HW) + xx[h];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int i = 2 * h + c;
            const int32_t q0 = acc[half][i], q1 = acc[2 + half][i], q2 = acc[4 + half][i], q3 = acc[6 + half][i];
            // conv1.cu's recombination: exact pairs, one fp32 rounding each, one FMA, the scale
            const float fu = (float)(q0 * 128 + q1);
            const float ft = (float)(q2 * 128 + q3);
            const int co = 8 * half + 2 * tig + c;
            ring[co * HW] = __fmaf_rn(ft, 1.0f / 16384.0f, fu) * s_scale[co];
          }
        }
      }
    }
    __syncthreads();
    // ---- pooled rows 3b .. 3b + 2 from conv rows 6b - 1 .. 6b + 5 ----
    for (int e = threadIdx.x; e < C_OUT * 3 * PHW; e += THREADS) {
      const int co = e / (3 * PHW), rem = e - co * (3 * PHW);
      const int py = 3 * b + rem / PHW, px = rem % PHW;
      float best = -INFINITY;
      int bi = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const int y = 2 * py - 1 + i;
        if (y < 0) continue;                                     // padded row (y <= 83 always)
        const float* ring = sRing + ((y + 1) % RING) * (C_OUT * HW) + co * HW;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const int x = 2 * px - 1 + j;
          if (x < 0) continue;                                   // padded column (x <= 83 always)
          const float v = ring[x];
          if (v > best || v != v) { best = v; bi = 3 * i + j; }  // first maximum, as max_pool2d (NaN wins)
        }
      }
      const int o = co * (PHW * PHW) + py * PHW + px;
      pooled[o] = best;
      if (ARGMAX) amax[o] = (uint8_t)bi;
    }
    __syncthreads();
  }
}

// this thread's A groups (c, ky): tig, tig + 4, tig + 8 -> byte offset of padded row ky of channel c
__device__ __forceinline__ void group_offsets(int tig, int (&goff)[3]) {
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int g = tig + 4 * q;
    goff[q] = (g / 3) * PAD_PLANE + (g % 3) * PAD_W;
  }
}

constexpr int PACK_BYTES = N_COLS * K_PAD;         // 3 072: one network's packed digits

struct PairParams {
  FrameSource src;
  const int64_t* idx;        // sampled rows, or nullptr for rows 0..n-1
  int64_t n;
  const int8_t* bq;          // [2][64][48]: net 0's pack, then net 1's
  const float* scale;        // [2][16]
  float* pooled;             // [2][n][16][42][42]
  uint8_t* argmax;           // net 0's [n][16][42][42] (ARGMAX only)
};

// Both networks' stems over the same rows (R2D2's online and target nets): each stack is loaded and zero-bordered
// once, then run through k_stem_fused's bands against net 0's digits and then net 1's, on the one ring (a second ring
// would not leave two CTAs per SM).  Per net the arithmetic is k_stem_fused's, so each net's output is bit for bit a
// single-net launch's with that net's pack.  ARGMAX: write net 0's argmax (net 1's is never needed).
template <FrameKind KIND, bool ARGMAX>
__global__ void __launch_bounds__(THREADS, 2)
k_stem_fused_pair(const __grid_constant__ PairParams P) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* sRaw = smem_raw;
  uint8_t* sPad = sRaw + RAW_BYTES;
  float* sRing = reinterpret_cast<float*>(sPad + PAD_BYTES);   // [7][16][84]: conv row r in slot (r + 1) % 7
  __shared__ __align__(8) uint64_t raw_full;
  __shared__ float s_scale[2 * C_OUT];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gid = lane >> 2, tig = lane & 3;
  if (threadIdx.x < 2 * C_OUT) s_scale[threadIdx.x] = P.scale[threadIdx.x] * (1.0f / 128.0f);   // exact
  zero_pad(sPad);
  if (threadIdx.x == 0) {
    mbar_init(&raw_full, 1);
    mbar_init_fence();
  }
  __syncthreads();
  const uint8_t* frames = frame_base<KIND>(P.src);
  if (threadIdx.x == 0 && blockIdx.x < P.n)
    load_row<KIND>(P.src, frames, clamp_row(P.src, P.idx, blockIdx.x), sRaw, &raw_full);
  int goff[3];
  group_offsets(tig, goff);

  int it = 0;
  for (int64_t k = blockIdx.x; k < P.n; k += gridDim.x, ++it) {
    mbar_wait(&raw_full, it & 1);
    fill_pad(sRaw, sPad);
    fence_async_smem();
    __syncthreads();
    if (threadIdx.x == 0 && k + gridDim.x < P.n)
      load_row<KIND>(P.src, frames, clamp_row(P.src, P.idx, k + gridDim.x), sRaw, &raw_full);
    // the fragments are reloaded per net (L1-resident 3 KB packs) rather than held for both: the same registers as
    // k_stem_fused
    uint32_t bw[8][3];
    load_weight_frags(P.bq, gid, tig, bw);
    conv_pool_stack<ARGMAX>(sPad, sRing, bw, goff, s_scale, P.pooled + k * POOLED, ARGMAX ? P.argmax + k * POOLED : nullptr,
                            warp, gid, tig);
    load_weight_frags(P.bq + PACK_BYTES, gid, tig, bw);
    conv_pool_stack<false>(sPad, sRing, bw, goff, s_scale + C_OUT, P.pooled + (P.n + k) * POOLED, nullptr, warp, gid,
                           tig);
  }
}

struct WgradParams {
  FrameSource src;
  const int64_t* idx;
  int64_t n;
  const float* gp;           // [n][16][42][42] dL/d(pooled)
  const uint8_t* argmax;     // [n][16][42][42]
  double* partial;           // [gridDim.x][16][36]
};

// gy of channel co at conv position (y, x): the pooled gradients whose window chose it, in (py, px) order
__device__ __forceinline__ float fold(const float* g, const uint8_t* a, int y, int x) {
  const int py0 = y >> 1, px0 = x >> 1;                    // window py covers rows 2py - 1 .. 2py + 1
  const int py1 = (y & 1) && py0 + 1 < PHW ? py0 + 1 : py0, px1 = (x & 1) && px0 + 1 < PHW ? px0 + 1 : px0;
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int py = i ? py1 : py0;
    if (i && py1 == py0) break;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int px = j ? px1 : px0;
      if (j && px1 == px0) break;
      const int o = py * PHW + px;
      if (a[o] == 3 * (y - 2 * py + 1) + (x - 2 * px + 1)) s = s + g[o];
    }
  }
  return s;
}

// digit scale of a channel: the power of two s = 2^(e-127) > absmax / 127 (conv1_wgrad.cu's digit_exponent)
__device__ __forceinline__ int digit_exponent(float absmax) {
  const float t = absmax / 127.0f;
  const int e = (int)((__float_as_uint(t) >> 23) & 0xFF) + 1;
  return e < 27 ? 27 : (e > 227 ? 227 : e);
}

template <FrameKind KIND>
__global__ void __launch_bounds__(THREADS, 1)
k_stem_wgrad(const __grid_constant__ WgradParams P) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* sRaw = smem_raw;
  uint8_t* sPad = sRaw + RAW_BYTES;
  float* sG = reinterpret_cast<float*>(sPad + PAD_BYTES);           // the stack's dL/dp [16][42][42]
  uint8_t* sA = reinterpret_cast<uint8_t*>(sG + POOLED);            // its argmax
  double* sRed = reinterpret_cast<double*>(sG);                     // [8 warps][16][36], after the last stack
  __shared__ __align__(8) uint64_t raw_full;
  __shared__ float s_wmax[WARPS][C_OUT];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gid = lane >> 2, tig = lane & 3;
  zero_pad(sPad);
  if (threadIdx.x == 0) {
    mbar_init(&raw_full, 1);
    mbar_init_fence();
  }
  __syncthreads();
  const uint8_t* frames = frame_base<KIND>(P.src);
  if (threadIdx.x == 0 && blockIdx.x < P.n)
    load_row<KIND>(P.src, frames, clamp_row(P.src, P.idx, blockIdx.x), sRaw, &raw_full);

  // B operand: patch element e = 8j + gid (c, ky, kx) of tile j, as a byte offset into the padded frame (-1: e >= 36)
  int eoff[E_TILES];
#pragma unroll
  for (int j = 0; j < E_TILES; ++j) {
    const int e = 8 * j + gid;
    eoff[j] = e < K_TAPS ? (e / 9) * PAD_PLANE + ((e % 9) / 3) * PAD_W + (e % 3) : -1;
  }
  double sum[E_TILES][4];
#pragma unroll
  for (int j = 0; j < E_TILES; ++j) sum[j][0] = sum[j][1] = sum[j][2] = sum[j][3] = 0.0;

  int it = 0;
  for (int64_t k = blockIdx.x; k < P.n; k += gridDim.x, ++it) {
    // ---- stage the stack's pooled gradient (with its per-channel max |.|) and argmax; the frames ----
    const float4* g4 = reinterpret_cast<const float4*>(P.gp + k * POOLED);
    float4* sG4 = reinterpret_cast<float4*>(sG);
#pragma unroll 1
    for (int co = 0; co < C_OUT; ++co) {
      float m = 0.0f;
      for (int i = threadIdx.x; i < PHW * PHW / 4; i += THREADS) {
        const float4 v = g4[co * (PHW * PHW / 4) + i];
        sG4[co * (PHW * PHW / 4) + i] = v;
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (lane == 0) s_wmax[warp][co] = m;
    }
    const uint4* a16 = reinterpret_cast<const uint4*>(P.argmax + k * POOLED);
    for (int i = threadIdx.x; i < POOLED / 16; i += THREADS) reinterpret_cast<uint4*>(sA)[i] = a16[i];
    mbar_wait(&raw_full, it & 1);
    fill_pad(sRaw, sPad);
    fence_async_smem();
    __syncthreads();
    if (threadIdx.x == 0 && k + gridDim.x < P.n)
      load_row<KIND>(P.src, frames, clamp_row(P.src, P.idx, k + gridDim.x), sRaw, &raw_full);

    // digit scales of this thread's channels gid and gid + 8: |folded gy| <= 4 max |dL/dp| (a rounded sum of at most
    // four terms never exceeds the exact bound, which is representable)
    float inv_s24[2], s_m24[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float m = 0.0f;
#pragma unroll
      for (int w = 0; w < WARPS; ++w) m = fmaxf(m, s_wmax[w][gid + 8 * h]);
      const int e = digit_exponent(4.0f * m);
      inv_s24[h] = __uint_as_float((uint32_t)(254 - e + 24) << 23);      // 2^24 / s
      s_m24[h] = __uint_as_float((uint32_t)(e - 24) << 23);              // s * 2^-24
    }

    int32_t acc[NSPLIT][E_TILES][4];
#pragma unroll
    for (int d = 0; d < NSPLIT; ++d)
#pragma unroll
      for (int j = 0; j < E_TILES; ++j) acc[d][j][0] = acc[d][j][1] = acc[d][j][2] = acc[d][j][3] = 0;

#pragma unroll 1
    for (int ks = warp; ks < K_STEPS; ks += WARPS) {
      // this thread's positions: p0 .. p0 + 3 (k bytes 4 tig ..) and p0 + 16 .. (k bytes 16 + 4 tig ..), each four in
      // one conv row (84 % 4 == 0); positions past 7 055 have gy = 0 and read row 0's pixels
      uint32_t a[NSPLIT][4];
      uint32_t b[E_TILES][2];
#pragma unroll
      for (int hp = 0; hp < 2; ++hp) {
        const int p = ks * 32 + 16 * hp + 4 * tig;
        const bool valid = p < POS;
        const int y = valid ? p / HW : 0, x0 = valid ? p - (p / HW) * HW : 0;
#pragma unroll
        for (int hc = 0; hc < 2; ++hc) {
          const int co = gid + 8 * hc;
          uint32_t Y[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float gy = valid ? fold(sG + co * (PHW * PHW), sA + co * (PHW * PHW), y, x0 + i) : 0.0f;
            // balanced base-256 digits via the bias 0x00808080 (conv1_wgrad.cu): low bytes q + 128, top byte q0
            Y[i] = (uint32_t)__float2int_rn(gy * inv_s24[hc]) + 0x00808080u;
          }
          const uint32_t t0 = __byte_perm(Y[0], Y[1], 0x5140), t1 = __byte_perm(Y[0], Y[1], 0x7362);
          const uint32_t t2 = __byte_perm(Y[2], Y[3], 0x5140), t3 = __byte_perm(Y[2], Y[3], 0x7362);
          // A fragment register: 0 (row gid, k lo), 1 (row gid + 8, k lo), 2 (row gid, k hi), 3 (row gid + 8, k hi)
          const int r = 2 * hp + hc;
          a[0][r] = __byte_perm(t1, t3, 0x7632);
          a[1][r] = __byte_perm(t1, t3, 0x5410) ^ 0x80808080u;
          a[2][r] = __byte_perm(t0, t2, 0x7632) ^ 0x80808080u;
          a[3][r] = __byte_perm(t0, t2, 0x5410) ^ 0x80808080u;
        }
        const uint8_t* prow = sPad + y * PAD_W + x0;
#pragma unroll
        for (int j = 0; j < E_TILES; ++j) b[j][hp] = eoff[j] >= 0 ? pad_word(prow, eoff[j]) : 0u;
      }
#pragma unroll
      for (int d = 0; d < NSPLIT; ++d)
#pragma unroll
        for (int j = 0; j < E_TILES; ++j) mma_k32_s8u8(acc[d][j], a[d], b[j][0], b[j][1]);
    }
    // the stack's exact digit sums -> int64 -> fp64 (exact: |X| < 7056 * 255 * 127 * 2^24 < 2^53), times s * 2^-24
#pragma unroll
    for (int j = 0; j < E_TILES; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const long long X = (((long long)acc[0][j][i] * 256 + acc[1][j][i]) * 256 + acc[2][j][i]) * 256 + acc[3][j][i];
        sum[j][i] += (double)X * (double)s_m24[i >> 1];
      }
    __syncthreads();               // every warp is done with sG, sA and sPad before the next stack is staged
  }

  // ---- per-warp sums -> SMEM, added in warp order; the CTA's partial ----
  // accumulator fragment: sum[j][2h + c] = row gid + 8h (channel), column 8j + 2 tig + c (patch element)
#pragma unroll
  for (int j = 0; j < E_TILES; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int co = gid + 8 * (i >> 1), e = 8 * j + 2 * tig + (i & 1);
      if (e < K_TAPS) sRed[(warp * C_OUT + co) * K_TAPS + e] = sum[j][i];
    }
  __syncthreads();
  for (int o = threadIdx.x; o < WG_OUT; o += THREADS) {
    double s = sRed[o];
#pragma unroll
    for (int w = 1; w < WARPS; ++w) s += sRed[w * WG_OUT + o];
    P.partial[(int64_t)blockIdx.x * WG_OUT + o] = s;
  }
}

// dW[i] (+)= (sum over CTAs of partial[cta][i], one fp64 sum in CTA order) / 255
__global__ void __launch_bounds__(WG_OUT / 2) k_stem_wgrad_reduce(const double* __restrict__ partial, int n_parts,
                                                                 int accumulate, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= WG_OUT) return;
  double s = 0.0;
#pragma unroll 8
  for (int p = 0; p < n_parts; ++p) s += partial[(int64_t)p * WG_OUT + i];   // the loads do not wait on the sum
  s = s / 255.0;
  out[i] = accumulate ? (float)((double)out[i] + s) : (float)s;
}

constexpr size_t FWD_SMEM = (size_t)RAW_BYTES + PAD_BYTES + RING_BYTES;                      // 96 192
constexpr size_t WGRAD_SMEM = (size_t)RAW_BYTES + PAD_BYTES + POOLED * 4 + POOLED;           // 199 680
static_assert(2 * (FWD_SMEM + 1024) <= 228 * 1024, "two forward CTAs per SM");
static_assert(WGRAD_SMEM + 1024 <= 227 * 1024, "stem wgrad shared memory");
static_assert((size_t)WARPS * WG_OUT * sizeof(double) <= POOLED * 4, "the warp sums fit where dL/dp was staged");

// Host: the sources the stem serves.  Ape-X's coded planes and its plane stride 8 (s / s' transition pairs) are not
// stacks of a rollout.
inline int check_stem_frames(const b2rl_frames* frames, FrameSource& src, FrameKind& kind) {
  if (const int rc = check_frames(frames, src, kind)) return rc;
  B2RL_REQUIRE(kind != FrameKind::CodedPlanes, "the stem does not read a coded frame pool (Ape-X's coded planes)");
  B2RL_REQUIRE(!(kind == FrameKind::Planes && src.plane_stride == 8),
               "the stem does not read plane_stride 8 (Ape-X's s / s' plane table)");
  return B2RL_OK;
}

}  // namespace stem
}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_stem_pack(const float* w_dev, int8_t* bq_out_dev, float* scale_out_dev, void* stream) {
  B2RL_REQUIRE(w_dev && bq_out_dev && scale_out_dev, "null argument");
  B2RL_REQUIRE((uintptr_t)bq_out_dev % 16 == 0, "packed weights must be 16-byte aligned");
  stem::k_stem_pack<<<stem::C_OUT, 64, 0, (cudaStream_t)stream>>>(w_dev, bq_out_dev, scale_out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_stem_fused(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const int8_t* bq_dev,
                               const float* scale_dev, float* pooled_out_dev, uint8_t* argmax_out_dev, void* stream) {
  B2RL_REQUIRE(n >= 0, "negative n");
  stem::FwdParams P{};
  FrameKind kind;
  if (const int rc = stem::check_stem_frames(frames, P.src, kind)) return rc;
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(bq_dev && scale_dev && pooled_out_dev && argmax_out_dev, "null argument");
  B2RL_REQUIRE((uintptr_t)bq_dev % 16 == 0, "packed weights must be 16-byte aligned");
  int dev = 0, sms = 0;
  B2RL_CUDA(cudaGetDevice(&dev));
  B2RL_CUDA(sm_count(dev, &sms));
  P.idx = idx_dev, P.n = n, P.bq = bq_dev, P.scale = scale_dev, P.pooled = pooled_out_dev, P.argmax = argmax_out_dev;
  const unsigned grid = (unsigned)(n < 2 * (int64_t)sms ? n : 2 * (int64_t)sms);
  cudaStream_t st = (cudaStream_t)stream;
  const cudaError_t e = with_frame_kind(kind, [&](auto K) {
    constexpr FrameKind KIND = decltype(K)::value;
    if constexpr (KIND == FrameKind::CodedPlanes) {
      return cudaErrorInvalidValue;                       // refused by check_stem_frames
    } else {
      cudaError_t r = set_max_dynamic_smem<stem::k_stem_fused<KIND>>(dev, stem::FWD_SMEM);
      if (r != cudaSuccess) return r;
      stem::k_stem_fused<KIND><<<grid, stem::THREADS, stem::FWD_SMEM, st>>>(P);
      return cudaSuccess;
    }
  });
  B2RL_CUDA(e);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_stem_fused_pair(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const int8_t* bq_dev,
                                    const float* scale_dev, float* pooled_out_dev, uint8_t* argmax_out_dev,
                                    void* stream) {
  B2RL_REQUIRE(n >= 0, "negative n");
  stem::PairParams P{};
  FrameKind kind;
  if (const int rc = stem::check_stem_frames(frames, P.src, kind)) return rc;
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(bq_dev && scale_dev && pooled_out_dev, "null argument");
  B2RL_REQUIRE((uintptr_t)bq_dev % 16 == 0, "packed weights must be 16-byte aligned");
  int dev = 0, sms = 0;
  B2RL_CUDA(cudaGetDevice(&dev));
  B2RL_CUDA(sm_count(dev, &sms));
  P.idx = idx_dev, P.n = n, P.bq = bq_dev, P.scale = scale_dev, P.pooled = pooled_out_dev, P.argmax = argmax_out_dev;
  const unsigned grid = (unsigned)(n < 2 * (int64_t)sms ? n : 2 * (int64_t)sms);
  cudaStream_t st = (cudaStream_t)stream;
  const cudaError_t e = with_frame_kind(kind, [&](auto K) {
    constexpr FrameKind KIND = decltype(K)::value;
    if constexpr (KIND == FrameKind::CodedPlanes) {
      return cudaErrorInvalidValue;                       // refused by check_stem_frames
    } else {
      if (argmax_out_dev) {
        cudaError_t r = set_max_dynamic_smem<stem::k_stem_fused_pair<KIND, true>>(dev, stem::FWD_SMEM);
        if (r != cudaSuccess) return r;
        stem::k_stem_fused_pair<KIND, true><<<grid, stem::THREADS, stem::FWD_SMEM, st>>>(P);
      } else {
        cudaError_t r = set_max_dynamic_smem<stem::k_stem_fused_pair<KIND, false>>(dev, stem::FWD_SMEM);
        if (r != cudaSuccess) return r;
        stem::k_stem_fused_pair<KIND, false><<<grid, stem::THREADS, stem::FWD_SMEM, st>>>(P);
      }
      return cudaSuccess;
    }
  });
  B2RL_CUDA(e);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int64_t b2rl_stem_wgrad_workspace_doubles(void) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (sm_count(dev, &sms) != cudaSuccess) return -1;
  return (int64_t)sms * stem::WG_OUT;
}

extern "C" int b2rl_stem_wgrad(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const float* gpooled_dev,
                               const uint8_t* argmax_dev, double* workspace_dev, float* gw_dev, int32_t accumulate,
                               void* stream) {
  B2RL_REQUIRE(n >= 1, "n must be positive");
  stem::WgradParams P{};
  FrameKind kind;
  if (const int rc = stem::check_stem_frames(frames, P.src, kind)) return rc;
  B2RL_REQUIRE(gpooled_dev && argmax_dev && workspace_dev && gw_dev, "null argument");
  B2RL_REQUIRE((uintptr_t)gpooled_dev % 16 == 0 && (uintptr_t)argmax_dev % 16 == 0,
               "the pooled gradient and the argmax must be 16-byte aligned");
  int dev = 0, sms = 0;
  B2RL_CUDA(cudaGetDevice(&dev));
  B2RL_CUDA(sm_count(dev, &sms));
  P.idx = idx_dev, P.n = n, P.gp = gpooled_dev, P.argmax = argmax_dev, P.partial = workspace_dev;
  const unsigned grid = (unsigned)(n < sms ? n : sms);
  cudaStream_t st = (cudaStream_t)stream;
  const cudaError_t e = with_frame_kind(kind, [&](auto K) {
    constexpr FrameKind KIND = decltype(K)::value;
    if constexpr (KIND == FrameKind::CodedPlanes) {
      return cudaErrorInvalidValue;
    } else {
      cudaError_t r = set_max_dynamic_smem<stem::k_stem_wgrad<KIND>>(dev, stem::WGRAD_SMEM);
      if (r != cudaSuccess) return r;
      stem::k_stem_wgrad<KIND><<<grid, stem::THREADS, stem::WGRAD_SMEM, st>>>(P);
      return cudaSuccess;
    }
  });
  B2RL_CUDA(e);
  count_launch();
  B2RL_CHECK_LAUNCH();
  stem::k_stem_wgrad_reduce<<<2, stem::WG_OUT / 2, 0, st>>>(workspace_dev, (int)grid, accumulate ? 1 : 0, gw_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}
