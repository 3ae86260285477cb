// The 3xTF32 operand image of csrc/gemm.cu: what k_gemm_tf32x3 reads, and what every kernel that writes such an
// image (the packs in gemm.cu, the fused optimizer in optim.cu that keeps the dense heads' weight images current)
// must produce bit for bit.
//
// Layout: [term 0=hi,1=lo][k_chunk][row_tile][row_in_tile][128 B, 16-byte units XOR (row & 7)]
// tile_rows is 128 for the A (M) side and 256 for the B (N) side; a k_chunk is 32 floats of the contraction.
#pragma once
#include <cstdint>

namespace b2rl {
namespace image {

constexpr int KC = 32;                          // floats per K chunk (128 B)

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

// float offset of 16-byte unit `unit` (contraction elements 4 unit .. 4 unit + 3 of chunk kc) of image row `row`
__device__ __forceinline__ int64_t offset(int row, int kc, int unit, int tile_rows, int rows_pad) {
  const int rt = row / tile_rows, rr = row - rt * tile_rows;
  return (((int64_t)kc * (rows_pad / tile_rows) + rt) * tile_rows + rr) * KC + ((unit ^ (rr & 7)) << 2);
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
