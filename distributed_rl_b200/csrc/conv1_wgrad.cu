// Fused gather + weight gradient of the first convolution on the Hopper tensor cores (wgmma).
//
//   dW[co, c, ky, kx] = (1/255) * sum_{k, oy, ox} gy[k, oy, ox, co] * frame[idx[k]][c, 4oy+ky, 4ox+kx]
//
// the backward half of csrc/conv1.cu (baseline/baseNetwork.py:165-172; loss.backward() of
// APE_X/Learner.py:123-138).  The input of conv_1 is data, so only dL/dW is needed.  The unfused
// path gathers the sampled uint8 rows, converts them to fp32 NHWC (58 MB for a batch of 512) and runs
// cuDNN's fp32 wgrad; here the sampled rows go HBM -> SMEM (TMA bulk copy) -> transposed im2col
// (patch element x output position, uint8) -> wgmma -> registers, and are never staged in HBM.
//
// Arithmetic: the GEMM is D[e = (c,ky,kx)][co] = sum_p A[e][p] * G[co][p] with p = (k, oy, ox).
// A holds exact uint8 pixels, so the MMA runs on u8 x s8 -> s32.  The fp32 output gradient is written as
// four balanced base-256 digits (int8) against a per-(CTA, channel) power-of-two scale s > max|gy| / 127,
//     gy = s * (q0 + q1/2^8 + q2/2^16 + q3/2^24)     (exact for |gy| >= s, else rounded at s * 2^-24),
// the digits being four groups of C_OUT rows of the B operand (N = 4*C_OUT).  Integer accumulation over
// all of the CTA's frame stacks is exact; the epilogue recombines the digit sums pairwise in int64 with
// one fp32 rounding per pair, so every CTA partial is the sum of pixel x (32-bit fixed-point gy) to
// ~1 ulp.  Partials of the CTAs are summed in fp64 by k_conv1_wgrad_reduce (deterministic, no atomics).
//
// Warp roles per CTA (persistent, one CTA per SM, 16 warps):
//   warps 0-15    build one 128-position K chunk of both operands in SMEM, then each warpgroup issues the
//                 wgmma m64nNk32 of its 64 patch elements (M = 256 over four warpgroups) and builds the next
//                 chunk while they run; the accumulators stay in registers over all of the CTA's frame stacks
//     warps 0-7   A: SMEM frame -> [256 patch elements][128 positions] uint8, K-major SW128
//     warps 8-15  B: gy (NHWC fp32, global) -> digits -> [4*C_OUT][128 positions] int8
//                 (warp = 8 channels x half of a chunk's 16-position units); the ReLU mask of the CTA's first
//                 MASK_ITEMS items comes from shared memory, written by the pre-scan that finds the digit scale
//   thread 0 also issues the TMA bulk copy of the next frame stack when it starts on a stack's first chunk: the
//   buffer it overwrites was last read two stacks before, by chunks that every producer has finished
//
// A coded frame pool (FrameKind::CodedPlanes, b2rl_dedup_attach_coded): no TMA copy.  The A producers decode the
// frames (frame_codec.cuh) from global memory straight into the raw buffer, frame j of stack it + 1 after building
// chunk j of stack it, so the decoding fills the time the A producers would spend waiting for the B producers.  The
// per-chunk barrier that publishes a chunk also publishes the decoded frames; stack 0 is decoded before the loop.
#include "common.cuh"
#include "frames.cuh"
#include "hopper.cuh"

namespace b2rl {
namespace conv1w {

using namespace sm90;

constexpr int C_IN = 4, HW = 84, KS = 8, STRIDE = 4, OHW = 20;
constexpr int E_TOTAL = C_IN * KS * KS;            // 256 patch elements = GEMM M (four warpgroups of 64)
constexpr int RAW_STRIDE = 28288;
constexpr int POS = OHW * OHW;                     // 400 output positions per frame stack
constexpr int NSPLIT = 4;
constexpr int KCHUNK = 128;                        // positions per pipeline stage (one 128-byte K row)
constexpr int CHUNKS = 4;                          // 128 + 128 + 128 + 16 (+16 zero padding)
constexpr int A_BYTES = E_TOTAL * KCHUNK;          // 32 KiB
constexpr int STAGES = 3;                          // a stage is rebuilt two chunks after its MMAs were issued
constexpr int A_PRODUCERS = 256, B_PRODUCERS = 256;
constexpr int THREADS = A_PRODUCERS + B_PRODUCERS;
constexpr int MAX_ITEMS_PER_CTA = 160;             // int32 accumulators: 128*255*400*T < 2^31
// ReLU masks of a CTA's first MASK_ITEMS items kept on chip from the pre-scan (one word of channel bits per position),
// so the digit build does not read y again; 4 covers a batch of 512 on 132 SMs
constexpr int MASK_ITEMS = 4;

// byte offset of (row, 16-byte unit) in a one-chunk K-major SW128 operand
__device__ __forceinline__ int sw_row(int row) { return (row >> 3) * 1024 + (row & 7) * 128; }

struct Params {
  FrameSource src;           // where row r is read from (frames.cuh)
  const int64_t* idx;        // sampled rows, or nullptr for rows 0..n-1
  int64_t n;
  const float* gy;           // [n][400][C_OUT] fp32 (NHWC)
  const float* y;            // optional conv_1 output after ReLU, same layout: dL/dy is taken as gy * (y > 0); else nullptr
  float* partial;            // [gridDim.x][C_OUT][256]
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

// digit scale of channel co: the power of two s = 2^(e-127) > max|gy| / 127 (e clamped to [27, 227])
__device__ __forceinline__ int digit_exponent(uint32_t absmax_bits) {
  const float t = __uint_as_float(absmax_bits) / 127.0f;
  const int e = (int)((__float_as_uint(t) >> 23) & 0xFF) + 1;
  return e < 27 ? 27 : (e > 227 ? 227 : e);
}

template <int C_OUT, FrameKind KIND>
__global__ void __launch_bounds__(THREADS, 1)
k_conv1_wgrad(const __grid_constant__ Params P) {
  constexpr int N_TOTAL = NSPLIT * C_OUT;              // 128 (64 for 16 channels)
  constexpr int B_BYTES = N_TOTAL * KCHUNK;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (sptr(smem_raw) & 1023u)) & 1023u);
  uint8_t* sStage = smem;
  uint8_t* sZero = smem + STAGES * STAGE_BYTES;        // a B operand of zeros: the K steps past position 415
  uint8_t* sRaw = sZero + B_BYTES;
  uint32_t* sMask = reinterpret_cast<uint32_t*>(sRaw + 2 * RAW_STRIDE);   // [MASK_ITEMS][POS]: bit co is y > 0
  FcRows* sRows = reinterpret_cast<FcRows*>(sMask + MASK_ITEMS * POS);   // CodedPlanes: the decoders' row tables
  __shared__ __align__(8) uint64_t raw_full[2];
  __shared__ uint32_t s_absmax[32];                    // per channel: bits of max |gy| over this CTA's items

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < 32) s_absmax[threadIdx.x] = 0u;
  for (int i = threadIdx.x; i < B_BYTES / 16; i += THREADS) reinterpret_cast<uint4*>(sZero)[i] = make_uint4(0u, 0u, 0u, 0u);
  for (int i = threadIdx.x; i < MASK_ITEMS * POS; i += THREADS) sMask[i] = 0u;
  fence_async_smem();
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) mbar_init(&raw_full[i], 1);
    mbar_init_fence();
  }
  __syncthreads();
  const int64_t first = blockIdx.x, stride = gridDim.x;
  const uint8_t* frames = frame_base<KIND>(P.src);

  // frame stack `it` of this CTA -> raw buffer it & 1
  auto load_frame = [&](int64_t it) {
    const int64_t k = first + it * stride;
    if (k >= P.n) return;
    int64_t row = P.idx ? P.idx[k] : k;
    row = row < 0 ? 0 : (row >= P.src.rows ? P.src.rows - 1 : row);
    load_row<KIND>(P.src, frames, row, sRaw + (it & 1) * RAW_STRIDE, &raw_full[it & 1]);
  };
  // CodedPlanes: frame c of the CTA's stack `it` -> raw buffer it & 1, decoded by the eight A producer warps together
  auto decode = [&](int64_t it, int c) {
    const int64_t k = first + it * stride;
    if (k >= P.n) return;
    int64_t row = P.idx ? P.idx[k] : k;
    row = row < 0 ? 0 : (row >= P.src.rows ? P.src.rows - 1 : row);
    decode_frame<A_PRODUCERS / 32>(coded_frame(P.src, row, c), sRaw + (it & 1) * RAW_STRIDE + c * PLANE_BYTES,
                                   sRows, c & 1, 3, warp, lane);
  };
  if constexpr (KIND != FrameKind::CodedPlanes) {
    if (threadIdx.x == 0) load_frame(0);
  }

  const bool is_a = warp < A_PRODUCERS / 32;
  if constexpr (KIND == FrameKind::CodedPlanes) {
    if (is_a) {
      for (int c = 0; c < C_IN; ++c) decode(0, c);
      named_sync(3, A_PRODUCERS);
    }
  }
  // -------- the B producers first find max |gy| per channel over this CTA's items (the digit scale);
  //          the A producers need no scale and build the first chunk meanwhile --------
  if (!is_a) {
    const int pt = threadIdx.x - A_PRODUCERS;         // 0..255
    const int c4 = (pt * 4) % C_OUT;                  // this thread always sees channels c4..c4+3 (1024 % C_OUT == 0)
    uint4 m = make_uint4(0u, 0u, 0u, 0u);
    // last item first: the items the main loop starts with are then the ones most recently read, still in L2
    const int64_t last = first + (P.n - 1 - first) / stride * stride;
    for (int64_t k = last; k >= first; k -= stride) {
      const uint4* g = reinterpret_cast<const uint4*>(P.gy + k * (int64_t)(POS * C_OUT));
      const float4* yk = P.y ? reinterpret_cast<const float4*>(P.y + k * (int64_t)(POS * C_OUT)) : nullptr;
      const int64_t it = (k - first) / stride;
      uint32_t* mk = it < MASK_ITEMS ? sMask + it * POS : nullptr;
#pragma unroll
      for (int i = 0; i < (POS * C_OUT / 4 + 255) / 256; ++i) {
        const int e = pt + 256 * i;
        if (e < POS * C_OUT / 4) {
          uint4 v = g[e];
          if (yk) {                                    // ReLU mask of the fused forward
            const float4 yv = yk[e];
            v.x = yv.x > 0.0f ? v.x : 0u; v.y = yv.y > 0.0f ? v.y : 0u;
            v.z = yv.z > 0.0f ? v.z : 0u; v.w = yv.w > 0.0f ? v.w : 0u;
            const uint32_t bits = (yv.x > 0.0f ? 1u : 0u) | (yv.y > 0.0f ? 2u : 0u) | (yv.z > 0.0f ? 4u : 0u) |
                                  (yv.w > 0.0f ? 8u : 0u);
            if (mk && bits) atomicOr(&mk[4 * e / C_OUT], bits << c4);   // element 4e is position 4e / C_OUT
          }
          m.x = max(m.x, v.x & 0x7FFFFFFFu); m.y = max(m.y, v.y & 0x7FFFFFFFu);
          m.z = max(m.z, v.z & 0x7FFFFFFFu); m.w = max(m.w, v.w & 0x7FFFFFFFu);
        }
      }
    }
    atomicMax(&s_absmax[c4 + 0], m.x); atomicMax(&s_absmax[c4 + 1], m.y);
    atomicMax(&s_absmax[c4 + 2], m.z); atomicMax(&s_absmax[c4 + 3], m.w);
    named_sync(1, B_PRODUCERS);
  }

  // A producer mapping: warp aw = (c, ky) rows 4aw..4aw+3, lane = 4 consecutive positions
  const int aw = warp;
  // B producer mapping: channel group bw (8 channels), half uh of the chunk's 16-position units
  const int bw = (warp - A_PRODUCERS / 32) & 3, uh = (warp - A_PRODUCERS / 32) >> 2;
  const int c3 = lane & 7, pq = lane >> 3;
  const int co = 8 * bw + c3;
  const bool b_active = !is_a && (8 * bw) < C_OUT;
  float inv_s24 = 16777216.0f;
  if (b_active) inv_s24 = __uint_as_float((uint32_t)(254 - digit_exponent(s_absmax[co]) + 24) << 23);   // 2^24 / s

  // chunk `at` = (item at/4, chunk at%4); a B producer issues the loads of chunk at+1 before converting chunk at
  const int64_t n_items = (P.n - first + stride - 1) / stride;
  const int total = (int)n_items * CHUNKS;
  auto load_chunk = [&](int at, float (&v)[4][4]) {
    const int j = at & 3;
    const int64_t base = (first + (int64_t)(at >> 2) * stride) * (int64_t)(POS * C_OUT) + co;
    const float* g = P.gy + base;
    const int u0 = (j < CHUNKS - 1) ? uh * 4 : uh, nu = (j < CHUNKS - 1) ? 4 : 1;
#pragma unroll
    for (int uu = 0; uu < 4; ++uu) {
      const int p = j * KCHUNK + (u0 + uu) * 16 + 4 * pq;
#pragma unroll
      for (int i = 0; i < 4; ++i) v[uu][i] = (uu < nu && p < POS) ? g[(int64_t)(p + i) * C_OUT] : 0.0f;
    }
    if (P.y && (at >> 2) < MASK_ITEMS) {             // ReLU mask of the fused forward, kept by the pre-scan
      const uint32_t* mk = sMask + (at >> 2) * POS;
#pragma unroll
      for (int uu = 0; uu < 4; ++uu) {
        const int p = j * KCHUNK + (u0 + uu) * 16 + 4 * pq;
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (uu < nu && p < POS && !((mk[p + i] >> co) & 1u)) v[uu][i] = 0.0f;
      }
    } else if (P.y) {                                // later items: read y again
      const float* yk = P.y + base;
#pragma unroll
      for (int uu = 0; uu < 4; ++uu) {
        const int p = j * KCHUNK + (u0 + uu) * 16 + 4 * pq;
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (uu < nu && p < POS && !(yk[(int64_t)(p + i) * C_OUT] > 0.0f)) v[uu][i] = 0.0f;
      }
    }
  };
  float v[4][4], vn[4][4];
  if (b_active && total > 0) load_chunk(0, v);

  const int wg = warp >> 2;                          // this warpgroup's MMA rows: patch elements [64 wg, 64 wg + 64)
  Acc<N_TOTAL> acc;
  for (int at = 0; at < total; ++at) {
    const int stage = at % STAGES, j = at & 3;
    uint8_t* st = sStage + stage * STAGE_BYTES;
    if (is_a) {
      // ------------------- A: transposed im2col, uint8 -------------------
      const int it = at >> 2, s = it & 1;
      if constexpr (KIND != FrameKind::CodedPlanes) {
        if (j == 0) {
          if (threadIdx.x == 0) load_frame(it + 1);
          mbar_wait(&raw_full[s], (it >> 1) & 1);
        }
      }
      const uint8_t* raw = sRaw + s * RAW_STRIDE;
      const int p0 = j * KCHUNK + 4 * lane;          // this lane's 4 consecutive positions (same oy: 20 % 4 == 0)
      if (p0 < POS) {
        const int oy = p0 / OHW, ox0 = p0 - oy * OHW;
        const uint8_t* src0 = raw + (STRIDE * oy) * HW + STRIDE * ox0;
        const int unit = lane >> 2, word = (lane & 3) * 4;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int cy = aw * 4 + r;                 // (c, ky): 32 rows of 8 patch elements (kx = 0..7)
          const int c = cy >> 3, ky = cy & 7;
          const uint32_t* src = reinterpret_cast<const uint32_t*>(src0 + c * (HW * HW) + ky * HW);
          // pixels 4*ox0 .. 4*ox0+19: word i holds kx = 0..3 of position p0+i, word i+1 its kx = 4..7
          const uint32_t w0 = src[0], w1 = src[1], w2 = src[2], w3 = src[3], w4 = src[4];
          const int e0 = c * 64 + ky * 8;
          // 4x4 byte transposes: out[kx] = {w_a.b[kx], w_b.b[kx], w_c.b[kx], w_d.b[kx]} = positions p0..p0+3 of element kx
          const uint32_t t0 = __byte_perm(w0, w1, 0x5140), t1 = __byte_perm(w0, w1, 0x7362);
          const uint32_t t2 = __byte_perm(w2, w3, 0x5140), t3 = __byte_perm(w2, w3, 0x7362);
          const uint32_t u0 = __byte_perm(w1, w2, 0x5140), u1 = __byte_perm(w1, w2, 0x7362);
          const uint32_t u2 = __byte_perm(w3, w4, 0x5140), u3 = __byte_perm(w3, w4, 0x7362);
          const uint32_t o[8] = {__byte_perm(t0, t2, 0x5410), __byte_perm(t0, t2, 0x7632),
                                 __byte_perm(t1, t3, 0x5410), __byte_perm(t1, t3, 0x7632),
                                 __byte_perm(u0, u2, 0x5410), __byte_perm(u0, u2, 0x7632),
                                 __byte_perm(u1, u3, 0x5410), __byte_perm(u1, u3, 0x7632)};
#pragma unroll
          for (int kx = 0; kx < 8; ++kx) {           // row e0 + kx: (e & 7) == kx
            *reinterpret_cast<uint32_t*>(st + sw_row(e0 + kx) + ((unit ^ kx) << 4) + word) = o[kx];
          }
        }
      }
    } else {
      // ------------------- B: gy -> four signed 7-bit digits -------------------
      // this warp's units of the chunk: 4 of 8 (last chunk: unit 0 = positions 384..399, unit 1 = zeros)
      const int u0 = (j < CHUNKS - 1) ? uh * 4 : uh, nu = (j < CHUNKS - 1) ? 4 : 1;
      if (b_active && at + 1 < total) load_chunk(at + 1, vn);
      if (b_active) {
        uint8_t* dstB = st + A_BYTES;
#pragma unroll
        for (int uu = 0; uu < 4; ++uu) {
          if (uu >= nu) break;
          // X = gy / s * 2^24 as an int32 (exact: power-of-two scale, |X| <= 127 * 2^24); balanced base-256 digits
          // via the bias 0x00808080: the three low bytes come out as q + 128, the top byte is q0 itself.
          uint32_t Y[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) Y[i] = (uint32_t)__float2int_rn(v[uu][i] * inv_s24) + 0x00808080u;
          // 4x4 byte transpose: digit d of the four positions packed into one word
          const uint32_t t0 = __byte_perm(Y[0], Y[1], 0x5140), t1 = __byte_perm(Y[0], Y[1], 0x7362);
          const uint32_t t2 = __byte_perm(Y[2], Y[3], 0x5140), t3 = __byte_perm(Y[2], Y[3], 0x7362);
          const uint32_t d3 = __byte_perm(t0, t2, 0x5410) ^ 0x80808080u, d2 = __byte_perm(t0, t2, 0x7632) ^ 0x80808080u;
          const uint32_t d1 = __byte_perm(t1, t3, 0x5410) ^ 0x80808080u, d0 = __byte_perm(t1, t3, 0x7632);
          const int off = (((u0 + uu) ^ c3) << 4) + pq * 4;    // rows d*C_OUT + co: (row & 7) == c3
          *reinterpret_cast<uint32_t*>(dstB + sw_row(0 * C_OUT + co) + off) = d0;
          *reinterpret_cast<uint32_t*>(dstB + sw_row(1 * C_OUT + co) + off) = d1;
          *reinterpret_cast<uint32_t*>(dstB + sw_row(2 * C_OUT + co) + off) = d2;
          *reinterpret_cast<uint32_t*>(dstB + sw_row(3 * C_OUT + co) + off) = d3;
        }
      }
#pragma unroll
      for (int uu = 0; uu < 4; ++uu)
#pragma unroll
        for (int i = 0; i < 4; ++i) v[uu][i] = vn[uu][i];
    }
    fence_async_smem();                              // generic-proxy writes -> visible to the tensor core
    // The chunk is complete once every producer is here.  Passing this barrier also means every warpgroup has
    // waited for the MMAs of chunk at - 2, which read the stage that chunk at + 1 will overwrite (STAGES = 3).
    named_sync(2, THREADS);
    const uint32_t a_base = sptr(st) + wg * (64 * 128), b_base = sptr(st + A_BYTES);
    // last chunk: positions 384..399 (+16 zeros) in K step 0; its other K steps multiply by the zero operand, which
    // keeps the wgmma sequence free of branches (a divergent path would serialize every wgmma of the kernel)
    const uint32_t b_tail = (j < CHUNKS - 1) ? b_base : sptr(sZero);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      acc.mma(make_desc(a_base + ks * 32), make_desc((ks == 0 ? b_base : b_tail) + ks * 32), (at | ks) ? 1u : 0u);
    wg_commit();
    wg_wait<1>();
    if constexpr (KIND == FrameKind::CodedPlanes) {
      // frame j of the next stack, while this chunk's MMAs run; buffer (it + 1) & 1 was last read for stack it - 1,
      // before the barrier of this stack's chunk 0, and the barrier after the last frame publishes the stack
      if (is_a) {
        const int64_t it = at >> 2;
        decode(it + 1, j);
        if (j == CHUNKS - 1) named_sync(3, A_PRODUCERS);
      }
    }
  }
  wg_wait<0>();
  wg_fence_regs(acc.d);

  // ------------------------------- epilogue -------------------------------
  // fragment (hopper.cuh): patch elements e and e + 8, columns 8j + 2(lane % 4) + {0, 1}; column d * C_OUT + co is
  // digit d of channel co
  if (total == 0) return;
  float* out = P.partial + (int64_t)blockIdx.x * (C_OUT * E_TOTAL);
  const int e_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int jj = 0; jj < C_OUT / 8; ++jj) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int cc = 8 * jj + 2 * (lane & 3) + c;
      const float scale = __uint_as_float((uint32_t)(digit_exponent(s_absmax[cc]) - 8) << 23) / 255.0f;   // s * 2^-8 / 255
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = 4 * jj + 2 * h + c;
        const int32_t q0 = acc.d[i], q1 = acc.d[i + C_OUT / 2], q2 = acc.d[i + C_OUT], q3 = acc.d[i + 3 * C_OUT / 2];
        // digit sums recombined pairwise in exact int64, one fp32 rounding per half, one FMA, the scale
        const float fu = (float)((long long)q0 * 256 + (long long)q1);
        const float ft = (float)((long long)q2 * 256 + (long long)q3);
        out[cc * E_TOTAL + e_base + 8 * h] = __fmaf_rn(ft, 1.0f / 65536.0f, fu) * scale;
      }
    }
  }
}

// dW[i] (+)= sum over CTAs of partial[cta][i] in fp64, fixed order (deterministic, no atomics).
// Block = 32 outputs x 8 slices of the partials: slice j adds partials j, j+8, ... (about 19 independent coalesced
// loads per thread instead of a 132-long chain: the kernel is L2-latency bound), then the 8 slices are added in order.
constexpr int RED_SLICES = 8;
__global__ void __launch_bounds__(32 * RED_SLICES)
k_conv1_wgrad_reduce(const float* __restrict__ partial, int n_parts, int numel, int accumulate, float* __restrict__ out) {
  __shared__ double s_part[RED_SLICES][32];
  const int i = blockIdx.x * 32 + threadIdx.x, j = threadIdx.y;
  double s0 = 0.0, s1 = 0.0;
  if (i < numel) {
    int p = j;
    for (; p + RED_SLICES < n_parts; p += 2 * RED_SLICES) {
      s0 += (double)partial[(int64_t)p * numel + i];
      s1 += (double)partial[(int64_t)(p + RED_SLICES) * numel + i];
    }
    if (p < n_parts) s0 += (double)partial[(int64_t)p * numel + i];
  }
  s_part[j][threadIdx.x] = s0 + s1;
  __syncthreads();
  if (j == 0 && i < numel) {
    double s = s_part[0][threadIdx.x];
#pragma unroll
    for (int q = 1; q < RED_SLICES; ++q) s += s_part[q][threadIdx.x];
    out[i] = accumulate ? (float)((double)out[i] + s) : (float)s;
  }
}

template <int C_OUT, FrameKind KIND>
constexpr size_t smem_bytes() {
  return (size_t)STAGES * (A_BYTES + NSPLIT * C_OUT * KCHUNK) + 2 * (size_t)RAW_STRIDE + NSPLIT * C_OUT * KCHUNK + 1024 +
         (size_t)MASK_ITEMS * POS * sizeof(uint32_t) + (KIND == FrameKind::CodedPlanes ? DECODE_TABLES * sizeof(FcRows) : 0);
}
// the largest instance and the kernel's 1 KiB of static shared memory within the 227 KiB a CTA can have
static_assert(smem_bytes<32, FrameKind::CodedPlanes>() + 1024 <= 227 * 1024, "conv_1 wgrad shared memory");

}  // namespace conv1w
}  // namespace b2rl

using namespace b2rl;

template <int C_OUT, FrameKind KIND>
static cudaError_t wgrad_launch(const conv1w::Params& P, unsigned grid, cudaStream_t st) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess)
    e = set_max_dynamic_smem<conv1w::k_conv1_wgrad<C_OUT, KIND>>(dev, conv1w::smem_bytes<C_OUT, KIND>());
  if (e != cudaSuccess) return e;
  conv1w::k_conv1_wgrad<C_OUT, KIND><<<grid, conv1w::THREADS, conv1w::smem_bytes<C_OUT, KIND>(), st>>>(P);
  return cudaSuccess;
}

extern "C" int64_t b2rl_conv1_wgrad_workspace_floats(int32_t c_out) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (sm_count(dev, &sms) != cudaSuccess) return -1;
  return (int64_t)sms * c_out * conv1w::E_TOTAL;
}

extern "C" int b2rl_conv1_wgrad(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const float* gy_dev,
                                const float* y_relu_dev, int32_t c_out, float* workspace_dev, float* gw_dev,
                                int32_t accumulate, void* stream) {
  B2RL_REQUIRE(n >= 1, "n must be positive");
  FrameSource src;
  FrameKind kind;
  if (const int rc = check_frames(frames, src, kind)) return rc;
  B2RL_REQUIRE(gy_dev && workspace_dev && gw_dev, "null argument");
  B2RL_REQUIRE(c_out == 16 || c_out == 32, "c_out must be 16 or 32");
  B2RL_REQUIRE(((uintptr_t)gy_dev % 16 == 0) && ((uintptr_t)y_relu_dev % 16 == 0), "gy and y must be 16-byte aligned");
  int dev = 0;
  B2RL_CUDA(cudaGetDevice(&dev));
  int sms = 0;
  B2RL_CUDA(sm_count(dev, &sms));
  cudaStream_t st = (cudaStream_t)stream;
  const int numel = c_out * conv1w::E_TOTAL;
  const int64_t per_launch = (int64_t)sms * conv1w::MAX_ITEMS_PER_CTA;   // int32 accumulator bound
  for (int64_t off = 0; off < n; off += per_launch) {
    const int64_t m = (n - off < per_launch) ? n - off : per_launch;
    // without idx, launch j reads rows [off, off + m) of the source: its rows 0..m-1 once advanced by off
    const conv1w::Params P{idx_dev ? src : advance(src, kind, off), idx_dev ? idx_dev + off : nullptr, m,
                           gy_dev + off * (int64_t)(conv1w::POS * c_out),
                           y_relu_dev ? y_relu_dev + off * (int64_t)(conv1w::POS * c_out) : nullptr, workspace_dev};
    const unsigned grid = (unsigned)((m < sms) ? m : sms);
    const cudaError_t e = with_frame_kind(kind, [&](auto K) {
      constexpr FrameKind KIND = decltype(K)::value;
      return c_out == 32 ? wgrad_launch<32, KIND>(P, grid, st) : wgrad_launch<16, KIND>(P, grid, st);
    });
    B2RL_CUDA(e);
    count_launch();
    B2RL_CHECK_LAUNCH();
    conv1w::k_conv1_wgrad_reduce<<<(numel + 31) / 32, dim3(32, conv1w::RED_SLICES), 0, st>>>(
        workspace_dev, (int)grid, numel, (accumulate || off > 0) ? 1 : 0, gw_dev);
    count_launch();
    B2RL_CHECK_LAUNCH();
  }
  return B2RL_OK;
}
