// b2rl_uniform_fetch: the minibatch of IMPALA's captured in-process learner step (impala.Learner.fused_step with
// use_graph) in ONE launch.  The draw of b2rl_serve_fill_uniform (uniform.cuh) over the ring's valid region, written
// into the step's fixed buffers instead of a ring slot: idx, action / mu / reward time-major, done, and conv_1's
// time-major frame rows.  The frames themselves are not copied: conv_1 reads them in place in the replay payload, or
// for a frame-deduplicated rollout store (b2rl_dedup_attach_rollouts) through its plane table at stride 4, whose row
// numbering is the same.
//
// Replaces Replay.draw (torch.randperm on a torch generator) + DeviceReplay.gather of the small fields + the
// transposes and time_major_rows of impala.Learner.fused_step, whose host-side arguments a CUDA graph would bake in.
#include "tree.cuh"
#include "uniform.cuh"

namespace b2rl {

constexpr int FETCH_DRAWS = 32;      // draws per CTA
constexpr int FETCH_THREADS = 256;   // threads per CTA: the first FETCH_DRAWS draw, all of them copy

// CTA c draws [c * FETCH_DRAWS, ...) (one thread per draw, each writes its idx and scalars), then its threads copy the
// draws' rows of `steps` words time-major (dst[t * n + k]) and write their frame rows (row t * n + k of the frame
// table = idx[k] * (steps + 1) + t), both with consecutive threads on consecutive k.
__global__ void __launch_bounds__(FETCH_THREADS)
k_uniform_fetch(SmallFields small, const __grid_constant__ SmallRows rows, uint64_t* __restrict__ rng_state,
                int64_t n, int32_t steps, UniformDraw u, int64_t* __restrict__ idx_out,
                int64_t* __restrict__ frame_rows_out) {
  __shared__ int64_t s_row[FETCH_DRAWS];
  const int tid = threadIdx.x;
  uint64_t seed, offset;
  rng_stream_take(rng_state, n, seed, offset);      // every block, exactly as k_serve_fill_uniform
  const int64_t k0 = (int64_t)blockIdx.x * FETCH_DRAWS;
  const int64_t m = (n - k0 < FETCH_DRAWS) ? n - k0 : FETCH_DRAWS;
  if (tid < m) {
    uint32_t key[4];
    philox4x32_10(offset, seed, key);
    const int64_t k = k0 + tid;
    const int64_t j = uniform_row(u, key, k);
    s_row[tid] = j;
    idx_out[k] = j;
    fetch_small(small, j, k);
  }
  __syncthreads();
  for (int f = 0; f < rows.n; ++f)
    copy_small_rows_time_major(rows.f[f], [&](int64_t k) { return s_row[k - k0]; }, k0, k0 + m, n, tid,
                               FETCH_THREADS);
  if (frame_rows_out) {
    const int64_t S = steps + 1;
    for (int64_t i = tid; i < S * m; i += FETCH_THREADS) {
      const int64_t t = i / m, d = i - t * m;
      frame_rows_out[t * n + k0 + d] = s_row[d] * S + t;
    }
  }
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_uniform_fetch(b2rl_replay* h, int64_t n, int32_t steps, int64_t* idx_out_dev,
                                  void* const* fields_out_dev, int64_t* frame_rows_out_dev, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(idx_out_dev != nullptr, "null idx_out");
  B2RL_REQUIRE(n >= 1, "n must be >= 1");
  B2RL_REQUIRE(steps >= 1, "steps must be >= 1");
  const int64_t size = h->size;
  B2RL_REQUIRE(n <= size, "sample larger than population: n exceeds the stored records");
  B2RL_REQUIRE(size <= (1LL << 32), "a uniform draw is from at most 2^32 records");
  B2RL_REQUIRE(h->dedup == nullptr || dedup_rollout_stacks(h) == steps + 1,
               h->dedup == nullptr || dedup_rollout_stacks(h) == 0
                   ? "a frame-deduplicated replay of transitions or sequences holds no rollouts"
                   : "the rollout frame pool holds steps + 1 frame stacks per rollout: steps does not match it");
  SmallFields small{};
  SmallRows rows{};
  for (int f = 0; f < h->n_fields; ++f) {
    const int64_t b = h->field_bytes[f];
    uint8_t* out = fields_out_dev ? (uint8_t*)fields_out_dev[f] : nullptr;
    if (h->dedup != nullptr && f == dedup_planes_field(h)) {   // the rollout's stacks, read through its pool ids
      B2RL_REQUIRE(out == nullptr, "frames are read in place: a frame field takes frame rows, not a buffer");
      continue;
    }
    RolloutField kind;
    const char* bad = rollout_field(b, steps, kind);
    B2RL_REQUIRE(bad == nullptr, bad);
    if (kind == RolloutField::FRAMES) {
      B2RL_REQUIRE(out == nullptr, "frames are read in place: a frame field takes frame rows, not a buffer");
    } else if (out == nullptr) {
      continue;
    } else if (kind == RolloutField::STEPS) {
      rows.f[rows.n++] = SmallField{h->field[f], out, b};
    } else {
      small.src[small.n] = h->field[f];
      small.dst[small.n] = out;
      small.bytes[small.n] = (int)b;
      small.n++;
    }
  }
  const UniformDraw u = uniform_draw_over(size, h->head, h->capacity);
  DeviceGuard g(h->device);
  k_uniform_fetch<<<(unsigned)((n + FETCH_DRAWS - 1) / FETCH_DRAWS), FETCH_THREADS, 0, (cudaStream_t)stream>>>(
      small, rows, h->rng_dev, n, steps, u, idx_out_dev, frame_rows_out_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}
