// The 3xTF32 operand image of csrc/gemm.cu: what k_gemm_tf32x3 reads, and what every kernel that writes such an
// image (the packs in gemm.cu, the fused optimizer in optim.cu that keeps the dense heads' weight images current)
// must produce bit for bit.
//
// Layout: [term 0=hi,1=lo][k_half][row_tile][row_in_tile][64 B, 16-byte units XOR ((row >> 1) & 3)]
// tile_rows is 128 for the A (M) side and 256 for the B (N) side; a k_half is 16 floats of the contraction, so one
// {term, k_half, row_tile} tile is a whole SWIZZLE_64B K-major operand (8-row x 64-byte atoms, 512 B apart) and the
// GEMM's loader stages it with one bulk copy.  The contraction is padded to a multiple of KC = 32 floats (two
// halves), which is the unit the GEMM splits K by.
#pragma once
#include <cstdint>

namespace b2rl {
namespace image {

constexpr int KC = 32;                          // contraction padding and K-split unit (floats)
constexpr int KH = 16;                          // floats of one k_half (64 B rows)

// x = hi + lo, hi = rn_tf32(x), lo = x - hi (exact in fp32)
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  const uint32_t u = __float_as_uint(x);
  uint32_t h = (u + 0x1000u) & 0xFFFFE000u;                        // round to nearest on the 13 dropped bits
  if ((h & 0x7F800000u) == 0x7F800000u) h = u & 0xFFFFE000u;        // rounding reached inf (or x is inf/nan): truncate
  hi = __uint_as_float(h);
  lo = ((u & 0x7F800000u) == 0x7F800000u) ? 0.0f : x - hi;          // exact in fp32
  if ((u & 0x7F800000u) == 0x7F800000u) hi = x;
}

// floats between the hi and the lo image
__host__ __device__ __forceinline__ int64_t term_stride(int k_chunks, int rows_pad) {
  return (int64_t)k_chunks * rows_pad * KC;
}

// float offset of the 16-byte unit holding contraction elements k .. k + 3 (k a multiple of 4) of image row `row`
__device__ __forceinline__ int64_t offset(int row, int k, int tile_rows, int rows_pad) {
  const int rt = row / tile_rows, rr = row - rt * tile_rows;
  const int kh = k / KH, unit = (k / 4) & 3;
  return (((int64_t)kh * (rows_pad / tile_rows) + rt) * tile_rows + rr) * KH + ((unit ^ ((rr >> 1) & 3)) << 2);
}

// split v[0..3] and store the {hi, lo} units at `off` of an image with term stride `ts`
__device__ __forceinline__ void store_unit(float* __restrict__ img, int64_t off, int64_t ts, const float v[4]) {
  float hi[4], lo[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) split_tf32(v[e], hi[e], lo[e]);
  *reinterpret_cast<float4*>(img + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<float4*>(img + ts + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
}

}  // namespace image
}  // namespace b2rl
