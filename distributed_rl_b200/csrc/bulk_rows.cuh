// Row copies shared by k_gather_bulk (gather.cu) and k_serve_fill (serve.cu).  The TMA row copy: whole replay rows of
// the bulk fields go HBM -> SMEM -> HBM through the TMA engine's 1-D bulk copies, driven by one thread over a ring of
// shared-memory stages.  The SMs only issue descriptors; the payload never touches the register file.  Rows too
// small for it are copied in words by the other threads of the CTA (copy_small_rows, at the end).
//
// Work item = (draw k, field, chunk); a chunk is at most CHUNK bytes of one row, and items are numbered
// draw-major, then field, then chunk.  The driving thread keeps a ring of BULK_RING_BYTES / CHUNK stages:
//   load(item) : cp.async.bulk global -> smem, completes on mbarrier[stage]
//   store(item): cp.async.bulk smem -> global (bulk_group)
// and refills the stage of item t - LAG once all but the newest LAG store groups have finished reading SMEM.
#pragma once
#include "common.cuh"
#include "frames.cuh"
#include "hopper.cuh"

namespace b2rl {

constexpr int BULK_RING_BYTES = 229376;   // 224 KiB of dynamic shared memory per CTA; stages = BULK_RING_BYTES / CHUNK

// A field is copied as bulk rows when its row is at least 1 KiB and a whole number of 16-byte units (the
// granularity of a bulk copy); smaller rows cost more in descriptors than they move.
inline bool is_bulk_row(int64_t row_bytes) { return row_bytes >= 1024 && row_bytes % 16 == 0; }

struct BulkField {
  const uint8_t* src;   // replay field base
  uint8_t* dst;         // output base
  int64_t row_bytes;    // is_bulk_row
  int32_t chunks;       // ceil(row_bytes / CHUNK); time-major: steps * ceil(step_bytes / CHUNK)
  int32_t step_bytes;   // time-major destination only: bytes of one time step of the row (a multiple of 16)
  const int32_t* planes;   // plane rows only: chunk c of replay row `row` is pool frame planes[plane_stride row +
  int32_t plane_base;      // plane_base + c] (src is the frame pool), so a row of k frames is k PLANE_BYTES copies
  int32_t plane_stride;
};

struct BulkRows {
  BulkField f[B2RL_MAX_FIELDS];
  int64_t items_per_row;   // sum of chunks over the fields
  int32_t n;               // fields
  int32_t pad;

  void add(const uint8_t* src, uint8_t* dst, int64_t row_bytes, int chunk) {
    f[n] = BulkField{src, dst, row_bytes, (int32_t)((row_bytes + chunk - 1) / chunk), 0, nullptr, 0, 0};
    items_per_row += f[n].chunks;
    ++n;
  }
  // Rows of k frames assembled from a frame pool: output row k' is the frames of pool ids plane_base .. plane_base +
  // k - 1 of replay row row_of(k'), whose ids start at planes + stride * row_of(k'); one chunk per frame (the copy
  // loop's CHUNK must be at least PLANE_BYTES).  Ape-X: k = 4 at stride 8 (s: base 0, s': base 4); R2D2 strip
  // records: k = stride = T + 3, base 0.
  void add_planes(const uint8_t* pool, const int32_t* planes, int32_t stride, int32_t plane_base, int32_t k,
                  uint8_t* dst) {
    f[n] = BulkField{pool, dst, (int64_t)k * PLANE_BYTES, k, 0, planes, plane_base, stride};
    items_per_row += k;
    ++n;
  }
  // The time-major form of add_planes for rows of `steps` frame stacks (IMPALA rollout records, stride = 4 steps):
  // stack t of draw k, pool ids planes[stride row_of(k) + 4t .. 4t + 3], goes to output row t * batch + k; one chunk
  // per frame.  Only for a TIME_MAJOR copy.
  void add_planes_time_major(const uint8_t* pool, const int32_t* planes, int32_t stride, int64_t steps, uint8_t* dst) {
    f[n] = BulkField{pool, dst, steps * STACK_BYTES, (int32_t)(4 * steps), STACK_BYTES, planes, 0, stride};
    items_per_row += f[n].chunks;
    ++n;
  }
  // A row of `steps` time steps whose step t of draw k goes to output row t * batch + k: chunked per step, so no
  // chunk straddles two steps and each one is a single bulk copy with a contiguous destination.
  void add_time_major(const uint8_t* src, uint8_t* dst, int64_t row_bytes, int64_t steps, int chunk) {
    const int64_t step = row_bytes / steps;
    f[n] = BulkField{src, dst, row_bytes, (int32_t)(steps * ((step + chunk - 1) / chunk)), (int32_t)step, nullptr, 0,
                     0};
    items_per_row += f[n].chunks;
    ++n;
  }
};

// Walks a contiguous range of items without divisions; `row` is the replay row of draw k.  TIME_MAJOR: the
// destination of step t of draw k is output row t * batch + k (BulkRows::add_time_major).
template <int CHUNK, bool TIME_MAJOR = false>
struct ItemCursor {
  int64_t k, row;
  int32_t f, c;
  template <class RowOf>
  __device__ __forceinline__ void init(const BulkRows& T, const RowOf& row_of, int64_t item) {
    k = item / T.items_per_row;
    int32_t r = (int32_t)(item - k * T.items_per_row);
    f = 0;
    while (r >= T.f[f].chunks) { r -= T.f[f].chunks; ++f; }
    c = r;
    row = row_of(k);
  }
  __device__ __forceinline__ void get(const BulkRows& T, int64_t dst_k0, const uint8_t*& src, uint8_t*& dst,
                                      uint32_t& bytes, int64_t batch = 0) const {
    if (TIME_MAJOR && T.f[f].planes != nullptr) {   // frame c of the row is frame c % 4 of stack c / 4
      bytes = PLANE_BYTES;
      src = plane_ptr(T.f[f].src, T.f[f].planes, row, T.f[f].plane_stride, T.f[f].plane_base, c);
      dst = T.f[f].dst + ((int64_t)(c >> 2) * batch + dst_k0 + k) * STACK_BYTES + (int64_t)(c & 3) * PLANE_BYTES;
      return;
    }
    if (TIME_MAJOR) {
      const int32_t step = T.f[f].step_bytes;
      const int32_t cps = (step + CHUNK - 1) / CHUNK;   // chunks per step
      const int32_t t = c / cps;
      const int64_t off = (int64_t)(c - t * cps) * CHUNK;
      const int64_t rem = step - off;
      bytes = (uint32_t)(rem < CHUNK ? rem : CHUNK);
      src = T.f[f].src + row * T.f[f].row_bytes + (int64_t)t * step + off;
      dst = T.f[f].dst + ((int64_t)t * batch + dst_k0 + k) * step + off;
      return;
    }
    if (T.f[f].planes != nullptr) {
      bytes = PLANE_BYTES;
      src = plane_ptr(T.f[f].src, T.f[f].planes, row, T.f[f].plane_stride, T.f[f].plane_base, c);
      dst = T.f[f].dst + (dst_k0 + k) * T.f[f].row_bytes + (int64_t)c * PLANE_BYTES;
      return;
    }
    const int64_t off = (int64_t)c * CHUNK;
    const int64_t rem = T.f[f].row_bytes - off;
    bytes = (uint32_t)(rem < CHUNK ? rem : CHUNK);
    src = T.f[f].src + row * T.f[f].row_bytes + off;
    dst = T.f[f].dst + (dst_k0 + k) * T.f[f].row_bytes + off;
  }
  template <class RowOf>
  __device__ __forceinline__ void next(const BulkRows& T, const RowOf& row_of, bool more) {
    if (++c == T.f[f].chunks) {
      c = 0;
      if (++f == T.n) {
        f = 0;
        ++k;
        if (more) row = row_of(k);
      }
    }
  }
};

// Run by ONE thread of the CTA, which needs BULK_RING_BYTES of dynamic shared memory: copies items
// [first, first + items) of table T (items >= 1).  Draw k reads replay row row_of(k) and writes output row
// dst_k0 + k, or with TIME_MAJOR step t of it to output row t * batch + dst_k0 + k.
template <int CHUNK, int LAG, bool TIME_MAJOR = false, class RowOf>
__device__ __forceinline__ void copy_rows(const BulkRows& T, const RowOf& row_of, int64_t dst_k0, int64_t first,
                                          int64_t items, int64_t batch = 0) {
  constexpr int STAGES = BULK_RING_BYTES / CHUNK;
  static_assert(STAGES <= 32 && STAGES > LAG + 1, "ring geometry");
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar[STAGES];
  for (int s = 0; s < STAGES; ++s) sm90::mbar_init(&bar[s], 1);
  sm90::mbar_init_fence();

  uint32_t phase_bits = 0;  // bit s = parity to wait for on stage s
  ItemCursor<CHUNK, TIME_MAJOR> ld, stc;   // load cursor runs ahead of the store cursor
  ld.init(T, row_of, first);
  stc = ld;
  int64_t loaded = 0;
  // prologue: fill the ring
  const int64_t pre = items < STAGES ? items : STAGES;
  for (; loaded < pre; ++loaded) {
    const uint8_t* src; uint8_t* dst; uint32_t bytes;
    ld.get(T, dst_k0, src, dst, bytes, batch);
    sm90::mbar_expect_tx(&bar[loaded], bytes);
    sm90::bulk_g2s(smem + (size_t)loaded * CHUNK, src, bytes, &bar[loaded]);
    ld.next(T, row_of, loaded + 1 < items);
  }
  int s = 0;            // stage of item t
  int rs = 0;           // stage to recycle next (item t - LAG)
  for (int64_t t = 0; t < items; ++t) {
    const uint8_t* src; uint8_t* dst; uint32_t bytes;
    stc.get(T, dst_k0, src, dst, bytes, batch);
    sm90::mbar_wait(&bar[s], (phase_bits >> s) & 1u);
    phase_bits ^= (1u << s);
    sm90::bulk_s2g(dst, smem + (size_t)s * CHUNK, bytes);
    sm90::bulk_commit();
    stc.next(T, row_of, t + 1 < items);
    if (++s == STAGES) s = 0;
    // refill the stage used LAG items ago once its store has drained SMEM
    if (t >= LAG) {
      if (loaded < items) {
        sm90::bulk_wait_read<LAG>();   // all but the newest LAG store groups have finished reading SMEM
        const uint8_t* nsrc; uint8_t* ndst; uint32_t nbytes;
        ld.get(T, dst_k0, nsrc, ndst, nbytes, batch);
        sm90::mbar_expect_tx(&bar[rs], nbytes);
        sm90::bulk_g2s(smem + (size_t)rs * CHUNK, nsrc, nbytes, &bar[rs]);
        ++loaded;
        ld.next(T, row_of, loaded < items);
      }
      if (++rs == STAGES) rs = 0;
    }
  }
  sm90::bulk_wait_all();
}

// A field whose rows are neither bulk rows nor copied by the draw itself: copied by the CTA's threads in words.
struct SmallField {
  const uint8_t* src;   // field base
  uint8_t* dst;         // output base
  int64_t row_bytes;
};

// The small-row fields of one launch (R2D2's action and reward: 80 x 4 B; IMPALA's action, mu and reward: T x 4 B).
struct SmallRows {
  SmallField f[B2RL_MAX_FIELDS];
  int32_t n;
};

template <typename U, class RowOf>
__device__ __forceinline__ void copy_small_units(const U* __restrict__ src, U* __restrict__ dst, int64_t units_per_row,
                                                 const RowOf& row_of, int64_t k0, int64_t k1, int64_t u,
                                                 int64_t step) {
  for (u += k0 * units_per_row; u < k1 * units_per_row; u += step) {
    const int64_t k = u / units_per_row, w = u - k * units_per_row;
    dst[u] = src[row_of(k) * units_per_row + w];
  }
}

// Output rows [k0, k1) of a small field <- replay rows row_of(k), in 4-byte words when the row is a whole number of
// words, else in bytes.  The caller's threads take units u, u + step, ... of the range (shared by k_gather_bulk's
// warp 1 and k_serve_fill's warps 1..3).
template <class RowOf>
__device__ __forceinline__ void copy_small_rows(const SmallField& f, const RowOf& row_of, int64_t k0, int64_t k1,
                                                int64_t u, int64_t step) {
  if ((f.row_bytes & 3) == 0)
    copy_small_units(reinterpret_cast<const uint32_t*>(f.src), reinterpret_cast<uint32_t*>(f.dst), f.row_bytes >> 2,
                     row_of, k0, k1, u, step);
  else
    copy_small_units(f.src, f.dst, f.row_bytes, row_of, k0, k1, u, step);
}

// The time-major form for a row of T 4-byte steps (IMPALA's action, mu, reward): dst[t * batch + k] =
// src[row_of(k) * T + t] for k in [k0, k1).  Each thread reads consecutive words of a row.
template <class RowOf>
__device__ __forceinline__ void copy_small_rows_time_major(const SmallField& f, const RowOf& row_of, int64_t k0,
                                                           int64_t k1, int64_t batch, int64_t u, int64_t step) {
  const uint32_t* __restrict__ src = reinterpret_cast<const uint32_t*>(f.src);
  uint32_t* __restrict__ dst = reinterpret_cast<uint32_t*>(f.dst);
  const int64_t T = f.row_bytes >> 2;
  for (u += k0 * T; u < k1 * T; u += step) {
    const int64_t k = u / T, t = u - k * T;
    dst[t * batch + k] = src[row_of(k) * T + t];
  }
}

}  // namespace b2rl
