// The uniform draw without replacement of IMPALA's replay (random.sample, baseline/utils.py:310-315), shared by the
// two kernels that draw rollouts: k_serve_fill_uniform (serve.cu) fills a served time-major minibatch slot and
// k_uniform_fetch (uniform.cu) fills the fixed buffers of the learner's captured in-process step.  From the same
// (seed, counter, size, head) both pick the same slots.
//
// Draw k of a call is slot (tail + pi(k)) mod capacity, where pi is a keyed pseudorandom permutation of [0, size): a
// 4-round balanced Feistel network on the smallest even bit width w >= 2 with 2^w >= size, cycle-walked into
// [0, size).  The round keys are the four words of ONE Philox4x32-10 block at the call's first counter, so a draw is
// a pure function of (seed, counter, k) and the draws of one call are distinct by construction.
#pragma once
#include "bulk_rows.cuh"

namespace b2rl {

struct UniformDraw {
  int64_t size;        // the valid region [tail, tail + size) mod capacity
  int64_t tail;
  int64_t capacity;
  int32_t half;        // w / 2
  uint32_t mask;       // 2^half - 1
};

// The draw over the valid region [head - size, head) of a ring of `capacity` slots, as impala.Replay.draw takes it
// (0 < size <= 2^32).
inline UniformDraw uniform_draw_over(int64_t size, int64_t head, int64_t capacity) {
  UniformDraw u{};
  u.size = size;
  u.capacity = capacity;
  u.tail = ((head - size) % capacity + capacity) % capacity;
  int w = 2;
  while ((1LL << w) < size) w += 2;
  u.half = w / 2;
  u.mask = (1u << u.half) - 1u;
  return u;
}

__host__ __device__ __forceinline__ uint32_t feistel4(uint32_t x, const uint32_t key[4], int half, uint32_t mask) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const uint32_t L = x >> half, R = x & mask;
    x = (R << half) | (L ^ (lowbias32(R ^ key[r]) & mask));
  }
  return x;
}

__device__ __forceinline__ int64_t uniform_row(const UniformDraw& u, const uint32_t key[4], int64_t k) {
  uint32_t y = feistel4((uint32_t)k, key, u.half, u.mask);
  while ((int64_t)y >= u.size) y = feistel4(y, key, u.half, u.mask);   // k < size: the walk ends on k's cycle
  const int64_t j = u.tail + (int64_t)y;
  return j >= u.capacity ? j - u.capacity : j;
}

// The fields of a time-major rollout of `steps` steps (IMPALA/ReplayMemory.py:34-43, with steps = T): frames, a bulk
// row of steps + 1 equal steps (s_0 .. s_T); a row of `steps` 4-byte words (action, mu, reward); a 1/2/4/8-byte
// scalar (done).
enum class RolloutField { FRAMES, STEPS, SCALAR };

// nullptr and the kind of a field of `row_bytes`, or why such a field cannot be part of a time-major rollout.
inline const char* rollout_field(int64_t row_bytes, int32_t steps, RolloutField& kind) {
  if (is_bulk_row(row_bytes)) {
    kind = RolloutField::FRAMES;
    if (row_bytes % (steps + 1) == 0 && (row_bytes / (steps + 1)) % 16 == 0) return nullptr;
    return "a bulk row of a time-major rollout must be steps + 1 rows of a multiple of 16 bytes";
  }
  if (row_bytes == 4 * (int64_t)steps) {
    kind = RolloutField::STEPS;
    return nullptr;
  }
  if (row_bytes == 1 || row_bytes == 2 || row_bytes == 4 || row_bytes == 8) {
    kind = RolloutField::SCALAR;
    return nullptr;
  }
  return "a time-major rollout holds bulk rows of steps + 1 steps, rows of steps 4-byte words and 1/2/4/8-byte "
         "scalars only";
}

}  // namespace b2rl
