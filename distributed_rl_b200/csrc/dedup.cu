// Frame-deduplicated stores: ingest (hash -> resolve -> assign + copy) into a frame pool, and the bookkeeping of
// its eviction rule (include/b2rl.h b2rl_dedup_*, DESIGN.md §4.16, §4.18).
//
// A pushed batch of n records is R n frames, R frames per record, laid out as the batch's Layout says:
//   Pairs   Ape-X transitions, R = 8: frame j is plane j % 8 of record j / 8 (planes 0-3 of s, then of s')
//   Strips  R2D2 frame strips, R = T + 3: frame j is the contiguous strips' frame j, of record j / R; and IMPALA
//           rollouts (b2rl_dedup_attach_rollouts), R = 4 (T + 1): a rollout's `state` row is its T + 1 frame stacks
//           back to back, so it is a strip of R frames whose stack t is frames 4t .. 4t + 3 (DESIGN.md §4.20)
// and frame j % R of record r gets its pool id in planes[R slot(r) + j % R].
//   1. k_dedup_hash   one warp per frame: 64-bit content key, inserted into a batch table keyed by it that keeps the
//                     lowest position holding each key
//   2. k_dedup_resolve one warp per frame: a frame equal (all 7 056 bytes) to the lowest position with its key reuses
//                     it; any other frame probes the key table, whose entry for a key is the newest stored frame with
//                     that key, and reuses that frame when it lies inside the window and all its bytes are equal
//   3. k_dedup_scan   the remaining frames (misses) get seq = head, head + 1, ... in batch order (one CTA)
//   4. the host reads the miss count (one synchronisation), zeroes the priorities of the slots the eviction rule
//      kills, then k_dedup_copy writes the R pool ids of every record, copies the misses into the pool and enters them
//      in the key table; the other fields and the priorities follow as for b2rl_replay_push.
// Everything a frame's id depends on is a function of the record stream (keys, positions, the window), so the ids
// can be checked against a CPU model (tests/dedup_model.py).
// A strip handle's pool may live in pinned, mapped host memory (b2rl_dedup_attach_strips_placed, DESIGN.md §4.19).
// The kernels are the same: k_dedup_resolve compares a hit's frame and k_dedup_copy stores the misses through the
// pool's device alias with plain 16-byte loads and stores, over PCIe, in order on the push's stream.  The key
// tables, pool_key and the batch scratch stay in HBM.
// A strip or Ape-X handle's pool may instead be a ring of P 16-byte units holding each frame losslessly encoded
// (b2rl_dedup_attach_strips_coded, b2rl_dedup_attach_coded, frame_codec.cuh, DESIGN.md §4.21, §4.22).  Frame seq's entry seq % F is then a descriptor
// (absolute unit offset, length) and the same ids name it.  The same kernels run with CODED set: k_dedup_resolve
// compares a hit's encoding with the frame by decoding it, and sizes the misses; k_coded_offsets lays them out in the
// unit ring (a frame never straddles its end); k_dedup_copy encodes them in place.  The readers decode each sampled
// slot's frames (k_decode_planes), and conv_1 decodes an Ape-X pool's frames on chip (frames.cuh,
// FrameKind::CodedPlanes); every one of them finds an id's encoding through fc_entry (frame_codec.cuh).  A rollout
// handle's pool is coded too (b2rl_dedup_attach_rollouts_coded, DESIGN.md §4.23): its learner step decodes each drawn
// rollout's distinct frames into a staged pool (k_stage_rollouts) that conv_1 reads as a raw one, and its served slots
// decode time-major (k_decode_planes with TIME_MAJOR).
#include "common.cuh"
#include "frame_codec.cuh"

#include <new>
#include <vector>

int b2rl_tree_update_impl(b2rl_replay* h, const int64_t* idx_dev, int64_t ring_start, const float* vals_dev,
                          float const_val, int64_t n, cudaStream_t st, bool publish_size_too);

namespace b2rl {

constexpr int DD_FRAME = 84 * 84;                 // 7 056 bytes per frame
constexpr int DD_STACK = 4 * DD_FRAME;            // 28 224 bytes per stack
constexpr int DD_WORDS = DD_FRAME / 8;            // 882
constexpr int DD_VEC = DD_FRAME / 16;             // 441
constexpr unsigned long long DD_EMPTY = ~0ULL;    // key of an unused table entry (keys are below 2^63)
constexpr unsigned long long DD_KEY_BITS = 0x7FFFFFFFFFFFFFFFULL;
constexpr int64_t DD_MAX_FRAMES = 65536;          // frames per push: the batch scratch (8192 Ape-X records)
constexpr int DD_THREADS = 256;                   // 8 frames per CTA

enum class Layout { Pairs, Strips };

struct DedupState {
  int32_t planes_field = -1;
  int32_t R = 8;                                  // frames per record
  Layout layout = Layout::Pairs;
  int32_t stacks = 0;                             // b2rl_dedup_attach_rollouts: frame stacks per rollout (T + 1)
  int64_t F = 0, W = 0, T = 0;                    // pool frames, window, key-table entries (a power of two)
  unsigned long long mask = 0;
  uint8_t* pool = nullptr;                        // [F][7056] the address kernels use: device memory, or the device
                                                  // alias of a host pool's pinned frames
  uint8_t* pool_host = nullptr;                   // b2rl_dedup_attach_strips_placed: the host address of a host pool
  unsigned long long* pool_key = nullptr;         // [F] key of the frame in each pool slot, for table rebuilds
  unsigned long long* tkey = nullptr;             // [T]
  unsigned long long* tseq = nullptr;             // [T] 1 + seq of the newest frame stored under tkey (0: none)
  int64_t used = 0;                               // table entries claimed since the last rebuild, at most
  int64_t head = 0;                               // frames stored so far
  int64_t max_batch = 0;
  int64_t BT = 0;                                 // batch-table entries (a power of two >= 2 R max_batch)
  unsigned long long* key = nullptr;              // [R max_batch] per batch frame
  int32_t* rep = nullptr;                         // [R max_batch] position whose frame it reuses (itself if none)
  int64_t* fseq = nullptr;                        // [R max_batch] seq (-1 before the scan: a miss)
  unsigned long long* bkey = nullptr;             // [BT]
  int32_t* bpos = nullptr;                        // [BT] lowest batch position holding bkey
  int64_t* misses_dev = nullptr;
  int64_t* misses_host = nullptr;                 // pinned
  cudaEvent_t done = nullptr;                     // recorded behind each push: the next one waits for it, so pushes
                                                  // on different streams never share the scratch or the key table
  std::vector<int64_t> ins;                       // per slot: head at the start of the batch that inserted it
  // b2rl_dedup_attach_strips_coded, _coded: pool is a ring of P 16-byte units of encoded frames, then FC_RAW_BYTES of
  // zeros
  int64_t P = 0;                                  // 0: frames stored raw, frame seq at pool + (seq % F) 7056
  int64_t units = 0;                              // units written so far, wrap padding included
  int64_t* foff = nullptr;                        // [F] absolute unit offset of the frame in each entry
  int32_t* flen = nullptr;                        // [F] its length in units
  int32_t* usz = nullptr;                         // [R max_batch] units of each miss's encoding
  int64_t* uoff = nullptr;                        // [R max_batch] absolute unit offset of each miss
  std::vector<int64_t> uins;                      // per slot: units at the start of the batch that inserted it
};

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {   // splitmix64's finaliser
  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ULL;
  z ^= z >> 27; z *= 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

// Frame j of the batch.  Pairs: plane j % 8 of record j / 8, from s and ns.  Strips: frame j of the strips s.
template <Layout L>
__device__ __forceinline__ const uint8_t* batch_frame(const uint8_t* s, const uint8_t* ns, int64_t j) {
  if constexpr (L == Layout::Strips) return s + j * DD_FRAME;
  const int64_t r = j >> 3;
  const int c = (int)(j & 7);
  return (c < 4 ? s : ns) + r * DD_STACK + (c & 3) * DD_FRAME;
}

__device__ __forceinline__ bool warp_equal(const uint8_t* a, const uint8_t* b, int lane) {
  const uint4* x = reinterpret_cast<const uint4*>(a);
  const uint4* y = reinterpret_cast<const uint4*>(b);
  bool eq = true;
  for (int i = lane; i < DD_VEC; i += 32) {
    const uint4 u = x[i], v = y[i];
    eq = eq && u.x == v.x && u.y == v.y && u.z == v.z && u.w == v.w;
  }
  return __all_sync(0xffffffffu, eq);
}

// Entry of `key` in an open-addressing table of `size` entries (claimed if absent).  The table never fills: the host
// keeps at most half of its entries claimed.
__device__ __forceinline__ int64_t claim(unsigned long long* keys, int64_t size, unsigned long long key) {
  int64_t i = (int64_t)(key & (unsigned long long)(size - 1));
  while (true) {
    const unsigned long long old = atomicCAS(keys + i, DD_EMPTY, key);
    if (old == DD_EMPTY || old == key) return i;
    i = (i + 1) & (size - 1);
  }
}

// Entry of `key`, or -1.
__device__ __forceinline__ int64_t find(const unsigned long long* keys, int64_t size, unsigned long long key) {
  int64_t i = (int64_t)(key & (unsigned long long)(size - 1));
  while (true) {
    const unsigned long long k = keys[i];
    if (k == key) return i;
    if (k == DD_EMPTY) return -1;
    i = (i + 1) & (size - 1);
  }
}

// key = mix64(sum over the frame's 8-byte words w_i of mix64(w_i ^ i * golden)) & mask, without its top bit.  The sum
// is order-free, so the lanes' partial sums combine in any order.
template <Layout L>
__global__ void __launch_bounds__(DD_THREADS)
k_dedup_hash(const uint8_t* __restrict__ s, const uint8_t* __restrict__ ns, int64_t frames, unsigned long long mask,
             unsigned long long* __restrict__ key, unsigned long long* __restrict__ bkey, int32_t* __restrict__ bpos,
             int64_t BT) {
  const int64_t j = ((int64_t)blockIdx.x * DD_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= frames) return;
  const uint64_t* w = reinterpret_cast<const uint64_t*>(batch_frame<L>(s, ns, j));
  uint64_t h = 0;
  for (int i = lane; i < DD_WORDS; i += 32) h += mix64(w[i] ^ ((uint64_t)i * 0x9E3779B97F4A7C15ULL));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  if (lane == 0) {
    const unsigned long long k = mix64(h) & mask & DD_KEY_BITS;
    key[j] = k;
    atomicMin(bpos + claim(bkey, BT, k), (int32_t)j);
  }
}

struct ResolveArgs {
  const uint8_t* s;
  const uint8_t* ns;
  int64_t frames;
  const unsigned long long* key;
  const unsigned long long* bkey;
  const int32_t* bpos;
  int64_t BT;
  const unsigned long long* tkey;
  const unsigned long long* tseq;
  int64_t T;
  const uint8_t* pool;
  int64_t F;
  int64_t oldest;           // head - W: the oldest seq a hit may reuse
  int32_t* rep;
  int64_t* fseq;
  int64_t P;                // a coded pool: units in the ring (a raw pool: 0, and the pointers below null)
  const int64_t* foff;
  int32_t* usz;             // a coded pool: units of each miss's encoding
};

// CODED: a hit's stored encoding is decoded and compared with the frame, and every miss gets the length of its
// encoding in usz.
template <Layout L, bool CODED>
__global__ void __launch_bounds__(DD_THREADS)
k_dedup_resolve(const __grid_constant__ ResolveArgs A) {
  const int64_t j = ((int64_t)blockIdx.x * DD_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= A.frames) return;
  const unsigned long long k = A.key[j];
  const uint8_t* me = batch_frame<L>(A.s, A.ns, j);
  const int32_t first = A.bpos[find(A.bkey, A.BT, k)];
  if (first < j && warp_equal(batch_frame<L>(A.s, A.ns, first), me, lane)) {
    if (lane == 0) { A.rep[j] = first; A.fseq[j] = -2; }
    return;
  }
  int64_t cand = -1;
  if (lane == 0) {
    const int64_t e = find(A.tkey, A.T, k);
    if (e >= 0) {
      const unsigned long long s1 = A.tseq[e];
      if (s1 > 0 && (int64_t)(s1 - 1) >= A.oldest) cand = (int64_t)(s1 - 1);
    }
  }
  cand = __shfl_sync(0xffffffffu, cand, 0);
  bool hit;
  int units = 0;
  if constexpr (CODED) {
    __shared__ FcRows s_rows[DD_THREADS / 32];
    hit = cand >= 0 && fc_equal(fc_entry(A.pool, A.P, A.foff, A.F, (int32_t)(cand % A.F)), me, s_rows[threadIdx.x >> 5],
                                lane);
    units = hit ? 0 : fc_encode(me, nullptr, lane);
  } else {
    hit = cand >= 0 && warp_equal(A.pool + (cand % A.F) * DD_FRAME, me, lane);
  }
  if (lane == 0) {
    A.rep[j] = (int32_t)j;
    A.fseq[j] = hit ? cand : -1;
    if constexpr (CODED) A.usz[j] = units;
  }
}

// Misses (fseq == -1) get seq head, head + 1, ... in batch order; *misses = their count.  One CTA of 1024 threads.
__global__ void __launch_bounds__(1024)
k_dedup_scan(int64_t* __restrict__ fseq, int64_t frames, int64_t head, int64_t* __restrict__ misses) {
  __shared__ int32_t s_warp[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t running = 0;
  for (int64_t base = 0; base < frames; base += 1024) {
    const int64_t j = base + threadIdx.x;
    const int32_t flag = (j < frames && fseq[j] == -1) ? 1 : 0;
    int32_t incl = flag;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int32_t w = s_warp[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t v = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += v;
      }
      s_warp[lane] = wi - w;          // exclusive prefix of the warp totals
    }
    __syncthreads();
    if (flag) fseq[j] = head + running + s_warp[warp] + incl - 1;
    const int32_t total = __shfl_sync(0xffffffffu, incl, 31);   // warp 31's inclusive total
    __syncthreads();
    if (warp == 31) s_warp[0] = s_warp[31] + total;
    __syncthreads();
    running += s_warp[0];
    __syncthreads();
  }
  if (threadIdx.x == 0) *misses = running;
}

struct CopyArgs {
  const uint8_t* s;
  const uint8_t* ns;
  int64_t frames;
  const unsigned long long* key;
  const int32_t* rep;
  const int64_t* fseq;
  int64_t head;             // first seq of this batch's misses
  uint8_t* pool;
  unsigned long long* pool_key;
  int64_t F;
  unsigned long long* tkey;
  unsigned long long* tseq;
  int64_t T;
  int32_t* planes;          // the replay's planes field
  int64_t slot0, capacity;  // record r goes to slot (slot0 + r) % capacity
  int32_t R;                // Strips: frames per record (Pairs: 8)
  int64_t P;                // a coded pool: units in the ring (a raw pool: 0, and the pointers below null)
  const int64_t* uoff;      // a coded pool: absolute unit offset and units of each miss (k_coded_offsets, resolve)
  const int32_t* usz;
  int64_t* foff;            // a coded pool: the descriptor of each entry
  int32_t* flen;
};

// CODED: each miss is encoded in place at its unit offset, and its entry gets the descriptor.
template <Layout L, bool CODED>
__global__ void __launch_bounds__(DD_THREADS)
k_dedup_copy(const __grid_constant__ CopyArgs A) {
  const int64_t j = ((int64_t)blockIdx.x * DD_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= A.frames) return;
  const int32_t r = A.rep[j];
  const int64_t sq = A.fseq[r];
  const int64_t ps = sq % A.F;
  if (lane == 0) {
    const int64_t R = L == Layout::Pairs ? 8 : A.R;
    const int64_t rec = L == Layout::Pairs ? j >> 3 : j / R;
    int64_t slot = A.slot0 + rec;
    if (slot >= A.capacity) slot -= A.capacity;
    A.planes[slot * R + (j - rec * R)] = (int32_t)ps;
  }
  if (r != j || sq < A.head) return;        // a batch duplicate or a hit: nothing to store
  if constexpr (CODED) {
    const int64_t off = A.uoff[j];
    fc_encode(batch_frame<L>(A.s, A.ns, j), A.pool + (off % A.P) * 16, lane);
    if (lane == 0) {
      A.foff[ps] = off;
      A.flen[ps] = A.usz[j];
    }
  } else {
    const uint4* src = reinterpret_cast<const uint4*>(batch_frame<L>(A.s, A.ns, j));
    uint4* dst = reinterpret_cast<uint4*>(A.pool + ps * DD_FRAME);
    for (int i = lane; i < DD_VEC; i += 32) dst[i] = src[i];
  }
  if (lane == 0) {
    const unsigned long long k = A.key[j];
    A.pool_key[ps] = k;
    atomicMax(A.tseq + claim(A.tkey, A.T, k), (unsigned long long)(sq + 1));
  }
}

// The key table from scratch: the frames with seq in [lo, hi), newest per key.
__global__ void __launch_bounds__(256)
k_dedup_rebuild(const unsigned long long* __restrict__ pool_key, int64_t F, int64_t lo, int64_t hi,
                unsigned long long* __restrict__ tkey, unsigned long long* __restrict__ tseq, int64_t T) {
  const int64_t q = lo + (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (q >= hi) return;
  atomicMax(tseq + claim(tkey, T, pool_key[q % F]), (unsigned long long)(q + 1));
}

// After k_dedup_scan: the misses (fseq >= head) get absolute unit offsets in batch order from U0 on, and out[1] = the
// units written once they are stored.  A miss that would straddle the ring's end starts at the next multiple of P
// instead, and the skipped units count as written.  The attach bounds a batch's units plus that padding by P, so at
// most one miss of a batch straddles.  One CTA of 1024 threads.
__global__ void __launch_bounds__(1024)
k_coded_offsets(const int64_t* __restrict__ fseq, const int32_t* __restrict__ usz, int64_t frames, int64_t head,
                int64_t U0, int64_t P, int64_t* __restrict__ uoff, int64_t* __restrict__ out) {
  __shared__ int32_t s_warp[32];
  __shared__ int32_t s_total, s_jstar;
  __shared__ int64_t s_pad;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t running = U0;
  for (int64_t base = 0; base < frames; base += 1024) {
    const int64_t j = base + threadIdx.x;
    const int32_t u = (j < frames && fseq[j] >= head) ? usz[j] : 0;
    int32_t incl = u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const int32_t w = s_warp[lane];
      int32_t wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t v = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += v;
      }
      s_warp[lane] = wi - w;          // exclusive prefix of the warp totals
      if (lane == 31) { s_total = wi; s_pad = 0; s_jstar = 1 << 30; }
    }
    __syncthreads();
    int64_t a = running + s_warp[warp] + incl - u;
    if (u > 0 && a % P + u > P) { s_pad = P - a % P; s_jstar = threadIdx.x; }
    __syncthreads();
    if (u > 0) uoff[j] = a + ((int)threadIdx.x >= s_jstar ? s_pad : 0);
    running += s_total + s_pad;
  }
  if (threadIdx.x == 0) out[1] = running;
}

// Frame c = j % R of draw k = j / R: slot clamp_row(idx[k])'s frame c, decoded from the pool.  One warp per frame.
// Strips: into dst + j * 7 056, the (n, R, 84, 84) strips.  Pairs (R = 8): planes 0-3 into the (n, 4, 84, 84) s stacks
// at dst, planes 4-7 into the s' stacks at dst2; a NULL output's frames are skipped.  TIME_MAJOR (b2rl_serve_fill_uniform
// on a coded rollout handle, Strips with R = 4 (T + 1)): the destination of add_planes_time_major, frame c % 4 of row
// (c / 4) n + k of the (T + 1) n stacks at dst.
template <Layout L, bool TIME_MAJOR>
__global__ void __launch_bounds__(DD_THREADS)
k_decode_planes(const uint8_t* __restrict__ pool, int64_t P, const int64_t* __restrict__ foff, int64_t F,
                const int32_t* __restrict__ planes, int32_t R, const int64_t* __restrict__ idx, int64_t n,
                int64_t capacity, uint8_t* __restrict__ dst, uint8_t* __restrict__ dst2) {
  __shared__ FcRows s_rows[DD_THREADS / 32];
  const int64_t j = ((int64_t)blockIdx.x * DD_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n * R) return;
  const int64_t k = j / R;
  const int64_t c = j - k * R;
  uint8_t* out = dst + j * DD_FRAME;
  if constexpr (TIME_MAJOR) out = dst + (((c >> 2) * n + k) * 4 + (c & 3)) * DD_FRAME;
  if constexpr (L == Layout::Pairs) {
    out = (c < 4 ? dst : dst2);
    if (out == nullptr) return;
    out += (4 * k + (c & 3)) * DD_FRAME;
  }
  fc_decode(fc_entry(pool, P, foff, F, planes[R * clamp_row(idx[k], capacity) + c]), out, s_rows[threadIdx.x >> 5],
            lane);
}

// b2rl_dedup_stage_rollouts: frame c = j % R of draw k = j / R is pool id planes[R slot + c] % F of slot
// clamp_row(idx[k]).  staged_planes[j] = k R + i, i the first of the draw's R positions holding the same id, and only
// the warp of that first position decodes the frame, into staged_pool + (k R + c) 7 056.  The other staged frames are
// left as they were.  One warp per frame; the lanes compare 32 earlier positions at a time.
__global__ void __launch_bounds__(DD_THREADS)
k_stage_rollouts(const uint8_t* __restrict__ pool, int64_t P, const int64_t* __restrict__ foff, int64_t F,
                 const int32_t* __restrict__ planes, int32_t R, const int64_t* __restrict__ idx, int64_t n,
                 int64_t capacity, uint8_t* __restrict__ staged_pool, int32_t* __restrict__ staged_planes) {
  __shared__ FcRows s_rows[DD_THREADS / 32];
  const int64_t j = ((int64_t)blockIdx.x * DD_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n * R) return;
  const int64_t k = j / R;
  const int32_t c = (int32_t)(j - k * R);
  const int32_t* ids = planes + R * clamp_row(idx[k], capacity);
  const uint32_t id = (uint32_t)ids[c] % (uint32_t)F;   // fc_entry's entry
  int32_t first = c;
  for (int32_t i0 = 0; i0 < c; i0 += 32) {              // c is the warp's: every lane takes the same exit
    const int32_t i = i0 + lane;
    const unsigned m = __ballot_sync(0xffffffffu, i < c && (uint32_t)ids[i] % (uint32_t)F == id);
    if (m != 0u) {
      first = i0 + __ffs((int)m) - 1;
      break;
    }
  }
  if (lane == 0) staged_planes[j] = (int32_t)(k * R + first);
  if (first != c) return;
  fc_decode(fc_entry(pool, P, foff, F, ids[c]), staged_pool + j * DD_FRAME, s_rows[threadIdx.x >> 5], lane);
}

// b2rl_frame_encode / b2rl_frame_decode: frame j <-> the encoding at enc + j * FC_RAW_BYTES.  One warp per frame.
__global__ void __launch_bounds__(DD_THREADS)
k_frame_encode(const uint8_t* __restrict__ frames, int64_t n, uint8_t* __restrict__ enc, int32_t* __restrict__ units) {
  const int64_t j = ((int64_t)blockIdx.x * DD_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n) return;
  const int u = fc_encode(frames + j * DD_FRAME, enc + j * FC_RAW_BYTES, lane);
  if (lane == 0 && units != nullptr) units[j] = u;
}

__global__ void __launch_bounds__(DD_THREADS)
k_frame_decode(const uint8_t* __restrict__ enc, int64_t n, uint8_t* __restrict__ frames) {
  __shared__ FcRows s_rows[DD_THREADS / 32];
  const int64_t j = ((int64_t)blockIdx.x * DD_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n) return;
  fc_decode(enc + j * FC_RAW_BYTES, frames + j * DD_FRAME, s_rows[threadIdx.x >> 5], lane);
}

void dedup_free(b2rl_replay* h) {
  DedupState* d = h->dedup;
  if (d == nullptr) return;
  if (d->pool_host) cudaFreeHost(d->pool_host);
  else if (d->pool) cudaFree(d->pool);
  for (void* p : {(void*)d->pool_key, (void*)d->tkey, (void*)d->tseq, (void*)d->key, (void*)d->rep,
                  (void*)d->fseq, (void*)d->bkey, (void*)d->bpos, (void*)d->misses_dev, (void*)d->foff,
                  (void*)d->flen, (void*)d->usz, (void*)d->uoff})
    if (p) cudaFree(p);
  if (d->misses_host) cudaFreeHost(d->misses_host);
  if (d->done) cudaEventDestroy(d->done);
  delete d;
  h->dedup = nullptr;
}

int dedup_planes_field(const b2rl_replay* h) { return h->dedup->planes_field; }
const uint8_t* dedup_pool(const b2rl_replay* h) { return h->dedup->pool; }
int64_t dedup_pool_frames(const b2rl_replay* h) { return h->dedup->F; }
bool dedup_pool_on_host(const b2rl_replay* h) { return h->dedup->pool_host != nullptr; }
int dedup_strip_frames(const b2rl_replay* h) { return h->dedup->layout == Layout::Strips ? h->dedup->R : 0; }
int dedup_rollout_stacks(const b2rl_replay* h) { return h->dedup->stacks; }
bool dedup_pool_coded(const b2rl_replay* h) { return h->dedup->P > 0; }

static unsigned warps_grid(int64_t frames) { return (unsigned)((frames * 32 + DD_THREADS - 1) / DD_THREADS); }

// n draws' frames through k_decode_planes (one of its instantiations), one warp per frame.
template <class Kernel>
static int decode_planes(Kernel kernel, b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev,
                         uint8_t* dst2_dev, cudaStream_t st) {
  const DedupState* d = h->dedup;
  kernel<<<warps_grid(n * d->R), DD_THREADS, 0, st>>>(d->pool, d->P, d->foff, d->F,
                                                      (const int32_t*)h->field[d->planes_field], d->R, idx_dev, n,
                                                      h->capacity, dst_dev, dst2_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

int gather_coded_planes(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, uint8_t* dst2_dev,
                        cudaStream_t st) {
  const bool pairs = h->dedup->layout == Layout::Pairs;
  B2RL_REQUIRE((uintptr_t)dst_dev % 16 == 0 && (uintptr_t)dst2_dev % 16 == 0,
               pairs ? "frame stack outputs must be 16-byte aligned" : "frame strip outputs must be 16-byte aligned");
  B2RL_REQUIRE(pairs || dst2_dev == nullptr, "a strip handle has one frame output");
  if (n == 0 || (dst_dev == nullptr && dst2_dev == nullptr)) return B2RL_OK;
  return decode_planes(pairs ? k_decode_planes<Layout::Pairs, false> : k_decode_planes<Layout::Strips, false>, h,
                       idx_dev, n, dst_dev, dst2_dev, st);
}

int decode_rollouts_time_major(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* dst_dev, cudaStream_t st) {
  return decode_planes(k_decode_planes<Layout::Strips, true>, h, idx_dev, n, dst_dev, nullptr, st);
}

}  // namespace b2rl

using namespace b2rl;

static int64_t pow2_at_least(int64_t x) {
  int64_t p = 1024;
  while (p < x) p <<= 1;
  return p;
}

// b2rl_dedup_attach and _coded (Pairs, R = 8), b2rl_dedup_attach_strips, _placed and _strips_coded (Strips, R =
// frames_per_record).
// pool_bytes > 0: a coded pool of pool_bytes / 16 units.  The arguments are checked before the handle, so every
// refusal comes before any CUDA work.
static int dedup_attach(b2rl_replay* h, int32_t planes_field, Layout layout, int32_t R, int64_t pool_frames,
                        int64_t window, uint64_t hash_mask, bool pool_on_host, int64_t pool_bytes = 0) {
  B2RL_REQUIRE(!pool_on_host || layout == Layout::Strips,
               "an Ape-X (Pairs) frame pool stays in HBM: only a strip handle's pool can be placed on the host");
  B2RL_REQUIRE(pool_bytes == 0 || !pool_on_host, "a coded frame pool stays in HBM: it cannot be placed on the host");
  B2RL_REQUIRE(R >= 4 && R <= DD_MAX_FRAMES, "frames_per_record must be in [4, 65536]");
  B2RL_REQUIRE(window >= 0 && pool_frames - window > R,
               layout == Layout::Pairs ? "need window >= 0 and pool_frames - window > 8"
                                       : "need window >= 0 and pool_frames - window > frames_per_record");
  B2RL_REQUIRE(pool_frames < (1LL << 31), "pool_frames must be below 2^31");
  B2RL_REQUIRE(pool_bytes >= 0 && pool_bytes % 16 == 0, "pool_bytes must be a non-negative multiple of 16");
  B2RL_REQUIRE(pool_bytes == 0 || pool_bytes / 16 - (window + 2) * FC_RAW_UNITS >= (int64_t)R * FC_RAW_UNITS,
               layout == Layout::Pairs ? "need pool_bytes >= 7072 (window + 10): one record beyond the window"
                                       : "need pool_bytes >= 7072 (window + 2 + frames_per_record): one record beyond the window");
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(h->dedup == nullptr, "the replay already has a frame pool");
  B2RL_REQUIRE(!h->any_on_host, "a replay with fields placed on the host cannot take a frame pool");
  B2RL_REQUIRE(h->size == 0 && h->head == 0 && h->reserved == 0 && h->pipe_n == 0, "the replay must be empty");
  B2RL_REQUIRE(planes_field >= 0 && planes_field < h->n_fields && h->field_bytes[planes_field] == 4 * (int64_t)R,
               layout == Layout::Pairs ? "the planes field must hold 8 int32 per slot"
                                       : "the planes field must hold frames_per_record int32 per slot");
  DeviceGuard g(h->device);
  DedupState* d = new (std::nothrow) DedupState();
  if (!d) { set_error("out of host memory"); return B2RL_ERR_NOMEM; }
  h->dedup = d;
  d->planes_field = planes_field;
  d->R = R;
  d->layout = layout;
  d->F = pool_frames;
  d->W = window;
  d->mask = (unsigned long long)hash_mask;
  d->max_batch = (pool_frames - window - 1) / R;
  if (d->max_batch > DD_MAX_FRAMES / R) d->max_batch = DD_MAX_FRAMES / R;
  if (d->max_batch > h->capacity) d->max_batch = h->capacity;
  d->P = pool_bytes / 16;
  if (d->P > 0 && d->max_batch > (d->P - (window + 2) * FC_RAW_UNITS) / (R * (int64_t)FC_RAW_UNITS))
    d->max_batch = (d->P - (window + 2) * FC_RAW_UNITS) / (R * (int64_t)FC_RAW_UNITS);   // DESIGN.md §4.21
  const int64_t nf = R * d->max_batch;
  d->T = pow2_at_least(2 * (window + nf));   // at most half claimed: window + one batch
  d->BT = pow2_at_least(2 * nf);
  cudaError_t e = cudaSuccess;
  auto alloc = [&](void** p, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc(p, bytes);
  };
  if (pool_on_host) {   // pinned, mapped frames: the kernels read and write them through the device alias
    const size_t bytes = (size_t)d->F * DD_FRAME;
    const cudaError_t eh = cudaHostAlloc((void**)&d->pool_host, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
    if (eh != cudaSuccess) {
      d->pool_host = nullptr;
      set_error("cudaHostAlloc of %.3f GB (%zu bytes) of pinned host memory for a %lld-frame pool failed: %s",
                bytes * 1e-9, bytes, (long long)pool_frames, cudaGetErrorString(eh));
      dedup_free(h);
      cudaGetLastError();
      return B2RL_ERR_NOMEM;
    }
    e = cudaHostGetDevicePointer((void**)&d->pool, d->pool_host, 0);
  } else if (d->P > 0) {
    // FC_RAW_BYTES of slack past the ring: a decode reads at most that many bytes from a frame's start, whatever the
    // bytes there (fc_prepare), so a descriptor near the end of the ring never reads past the allocation.  Zeroed, so
    // an entry no frame has been written to decodes as an all-zero raw frame.
    alloc((void**)&d->pool, (size_t)d->P * 16 + FC_RAW_BYTES);
    if (e == cudaSuccess) e = cudaMemset(d->pool, 0, (size_t)d->P * 16 + FC_RAW_BYTES);
    alloc((void**)&d->foff, sizeof(int64_t) * (size_t)d->F);
    alloc((void**)&d->flen, sizeof(int32_t) * (size_t)d->F);
    alloc((void**)&d->usz, sizeof(int32_t) * (size_t)nf);
    alloc((void**)&d->uoff, sizeof(int64_t) * (size_t)nf);
    if (e == cudaSuccess) e = cudaMemset(d->foff, 0, sizeof(int64_t) * (size_t)d->F);
    if (e == cudaSuccess) e = cudaMemset(d->flen, 0, sizeof(int32_t) * (size_t)d->F);
  } else {
    alloc((void**)&d->pool, (size_t)d->F * DD_FRAME);
  }
  alloc((void**)&d->pool_key, sizeof(unsigned long long) * (size_t)d->F);
  alloc((void**)&d->tkey, sizeof(unsigned long long) * (size_t)d->T);
  alloc((void**)&d->tseq, sizeof(unsigned long long) * (size_t)d->T);
  alloc((void**)&d->key, sizeof(unsigned long long) * (size_t)nf);
  alloc((void**)&d->rep, sizeof(int32_t) * (size_t)nf);
  alloc((void**)&d->fseq, sizeof(int64_t) * (size_t)nf);
  alloc((void**)&d->bkey, sizeof(unsigned long long) * (size_t)d->BT);
  alloc((void**)&d->bpos, sizeof(int32_t) * (size_t)d->BT);
  alloc((void**)&d->misses_dev, 2 * sizeof(int64_t));        // misses, and units written (a coded pool)
  if (e == cudaSuccess) e = cudaMallocHost((void**)&d->misses_host, 2 * sizeof(int64_t));
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&d->done, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaMemset(d->tkey, 0xFF, sizeof(unsigned long long) * (size_t)d->T);
  if (e == cudaSuccess) e = cudaMemset(d->tseq, 0, sizeof(unsigned long long) * (size_t)d->T);
  if (e == cudaSuccess) e = cudaMemset(h->field[planes_field], 0, (size_t)h->capacity * 4 * R);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    if (d->P > 0)
      set_error("allocating a %lld-frame coded pool of %.3f GB failed: %s", (long long)pool_frames,
                pool_bytes * 1e-9, cudaGetErrorString(e));
    else
      set_error("allocating a %lld-frame pool failed: %s", (long long)pool_frames, cudaGetErrorString(e));
    dedup_free(h);
    cudaGetLastError();
    return B2RL_ERR_NOMEM;
  }
  try {
    d->ins.assign((size_t)h->capacity, 0);
    if (d->P > 0) d->uins.assign((size_t)h->capacity, 0);
  } catch (...) {
    dedup_free(h);
    set_error("out of host memory");
    return B2RL_ERR_NOMEM;
  }
  return B2RL_OK;
}

extern "C" int b2rl_dedup_attach(b2rl_replay* h, int32_t planes_field, int64_t pool_frames, int64_t window,
                                 uint64_t hash_mask) {
  return dedup_attach(h, planes_field, Layout::Pairs, 8, pool_frames, window, hash_mask, false);
}

extern "C" int b2rl_dedup_attach_strips(b2rl_replay* h, int32_t planes_field, int32_t frames_per_record,
                                        int64_t pool_frames, int64_t window, uint64_t hash_mask) {
  return dedup_attach(h, planes_field, Layout::Strips, frames_per_record, pool_frames, window, hash_mask, false);
}

extern "C" int b2rl_dedup_attach_strips_placed(b2rl_replay* h, int32_t planes_field, int32_t frames_per_record,
                                               int64_t pool_frames, int64_t window, uint64_t hash_mask,
                                               int32_t pool_on_host) {
  B2RL_REQUIRE(pool_on_host == 0 || pool_on_host == 1, "pool_on_host must be 0 or 1");
  return dedup_attach(h, planes_field, Layout::Strips, frames_per_record, pool_frames, window, hash_mask,
                      pool_on_host != 0);
}

extern "C" int b2rl_dedup_attach_strips_coded(b2rl_replay* h, int32_t planes_field, int32_t frames_per_record,
                                              int64_t pool_frames, int64_t window, uint64_t hash_mask,
                                              int64_t pool_bytes) {
  B2RL_REQUIRE(pool_bytes > 0, "pool_bytes must be positive");
  return dedup_attach(h, planes_field, Layout::Strips, frames_per_record, pool_frames, window, hash_mask, false,
                      pool_bytes);
}

extern "C" int b2rl_dedup_attach_coded(b2rl_replay* h, int32_t planes_field, int64_t pool_frames, int64_t window,
                                       uint64_t hash_mask, int64_t pool_bytes) {
  B2RL_REQUIRE(pool_bytes > 0, "pool_bytes must be positive");
  return dedup_attach(h, planes_field, Layout::Pairs, 8, pool_frames, window, hash_mask, false, pool_bytes);
}

// b2rl_dedup_attach_rollouts and _rollouts_coded: the strip attach with R = 4 stacks_per_record that marks the handle
// as holding rollouts.
static int rollout_attach(b2rl_replay* h, int32_t planes_field, int32_t stacks_per_record, int64_t pool_frames,
                          int64_t window, uint64_t hash_mask, int64_t pool_bytes) {
  B2RL_REQUIRE(stacks_per_record >= 1 && stacks_per_record <= DD_MAX_FRAMES / 4,
               "stacks_per_record must be in [1, 16384]");
  const int rc = dedup_attach(h, planes_field, Layout::Strips, 4 * stacks_per_record, pool_frames, window, hash_mask,
                              false, pool_bytes);
  if (rc == B2RL_OK) h->dedup->stacks = stacks_per_record;
  return rc;
}

extern "C" int b2rl_dedup_attach_rollouts(b2rl_replay* h, int32_t planes_field, int32_t stacks_per_record,
                                          int64_t pool_frames, int64_t window, uint64_t hash_mask) {
  return rollout_attach(h, planes_field, stacks_per_record, pool_frames, window, hash_mask, 0);
}

extern "C" int b2rl_dedup_attach_rollouts_coded(b2rl_replay* h, int32_t planes_field, int32_t stacks_per_record,
                                                int64_t pool_frames, int64_t window, uint64_t hash_mask,
                                                int64_t pool_bytes) {
  B2RL_REQUIRE(pool_bytes > 0, "pool_bytes must be positive");
  return rollout_attach(h, planes_field, stacks_per_record, pool_frames, window, hash_mask, pool_bytes);
}

extern "C" int b2rl_dedup_stage_rollouts(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* staged_pool_dev,
                                         int32_t* staged_planes_dev, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  const DedupState* d = h->dedup;
  B2RL_REQUIRE(d != nullptr && d->stacks > 0 && d->P > 0,
               "not a coded rollout frame pool (b2rl_dedup_attach_rollouts_coded)");
  B2RL_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(idx_dev != nullptr && staged_pool_dev != nullptr && staged_planes_dev != nullptr, "null argument");
  B2RL_REQUIRE((uintptr_t)staged_pool_dev % 16 == 0 && (uintptr_t)staged_planes_dev % 4 == 0,
               "the staged pool must be 16-byte aligned and the staged planes 4-byte aligned");
  B2RL_REQUIRE(n <= ((1LL << 31) - 1) / d->R, "n out of range: n * 4 (T + 1) staged frames must stay below 2^31");
  DeviceGuard g(h->device);
  k_stage_rollouts<<<warps_grid(n * d->R), DD_THREADS, 0, (cudaStream_t)stream>>>(
      d->pool, d->P, d->foff, d->F, (const int32_t*)h->field[d->planes_field], d->R, idx_dev, n, h->capacity,
      staged_pool_dev, staged_planes_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_dedup_info(const b2rl_replay* h, void** pool_dev, int64_t* head_seq, int64_t* max_batch) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(h->dedup != nullptr, "not a frame-deduplicated replay (b2rl_dedup_attach)");
  if (pool_dev) *pool_dev = h->dedup->pool;
  if (head_seq) *head_seq = h->dedup->head;
  if (max_batch) *max_batch = h->dedup->max_batch;
  return B2RL_OK;
}

extern "C" int b2rl_dedup_codec_stats(const b2rl_replay* h, int64_t* units_written, int64_t* pool_units,
                                      int64_t* frames_stored) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  B2RL_REQUIRE(h->dedup != nullptr && h->dedup->P > 0,
               "not a coded frame pool (b2rl_dedup_attach_strips_coded, _coded, _rollouts_coded)");
  if (units_written) *units_written = h->dedup->units;
  if (pool_units) *pool_units = h->dedup->P;
  if (frames_stored) *frames_stored = h->dedup->head;
  return B2RL_OK;
}

extern "C" int b2rl_dedup_coded_offsets(const b2rl_replay* h, void** offsets_dev) {
  B2RL_REQUIRE(h != nullptr && offsets_dev != nullptr, "null argument");
  B2RL_REQUIRE(h->dedup != nullptr && h->dedup->P > 0,
               "not a coded frame pool (b2rl_dedup_attach_strips_coded, b2rl_dedup_attach_coded)");
  *offsets_dev = h->dedup->foff;
  return B2RL_OK;
}

extern "C" int b2rl_frame_encode(const uint8_t* frames_dev, int64_t n, uint8_t* enc_dev, int32_t* units_dev,
                                 void* stream) {
  B2RL_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(frames_dev != nullptr && enc_dev != nullptr, "null argument");
  B2RL_REQUIRE((uintptr_t)frames_dev % 16 == 0 && (uintptr_t)enc_dev % 16 == 0, "buffers must be 16-byte aligned");
  k_frame_encode<<<warps_grid(n), DD_THREADS, 0, (cudaStream_t)stream>>>(frames_dev, n, enc_dev, units_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_frame_decode(const uint8_t* enc_dev, int64_t n, uint8_t* frames_dev, void* stream) {
  B2RL_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(frames_dev != nullptr && enc_dev != nullptr, "null argument");
  B2RL_REQUIRE((uintptr_t)frames_dev % 16 == 0 && (uintptr_t)enc_dev % 16 == 0, "buffers must be 16-byte aligned");
  k_frame_decode<<<warps_grid(n), DD_THREADS, 0, (cudaStream_t)stream>>>(enc_dev, n, frames_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_dedup_pool_placement(const b2rl_replay* h, int32_t* on_host, void** pool) {
  B2RL_REQUIRE(h != nullptr && on_host != nullptr, "null argument");
  B2RL_REQUIRE(h->dedup != nullptr, "not a frame-deduplicated replay (b2rl_dedup_attach)");
  *on_host = h->dedup->pool_host != nullptr ? 1 : 0;
  if (pool) *pool = *on_host ? h->dedup->pool_host : h->dedup->pool;
  return B2RL_OK;
}

// The push of n records whose frames the layout L places (the caller has checked the frame pointers).
template <Layout L>
static int dedup_push(b2rl_replay* h, const uint8_t* s_dev, const uint8_t* ns_dev, const void* const* fields_src,
                      const float* prios, int64_t n, cudaStream_t st) {
  DedupState* d = h->dedup;
  B2RL_REQUIRE(prios != nullptr && fields_src != nullptr, "null argument");
  B2RL_REQUIRE(fields_src[d->planes_field] == nullptr, "the planes field is written by the push itself");
  B2RL_REQUIRE(h->reserved == 0, "a reservation is pending");
  DeviceGuard g(h->device);
  const int64_t frames = d->R * n;
  const int64_t head = d->head;
  B2RL_CUDA(cudaStreamWaitEvent(st, d->done, 0));     // the previous push (on any stream) is done with the scratch
  // 1. the key table: rebuilt from the window when this batch could take it past half full
  if (d->used + frames > d->T / 2) {
    const int64_t lo = head > d->W ? head - d->W : 0;
    B2RL_CUDA(cudaMemsetAsync(d->tkey, 0xFF, sizeof(unsigned long long) * (size_t)d->T, st));
    B2RL_CUDA(cudaMemsetAsync(d->tseq, 0, sizeof(unsigned long long) * (size_t)d->T, st));
    if (head > lo) {
      k_dedup_rebuild<<<(unsigned)((head - lo + 255) / 256), 256, 0, st>>>(d->pool_key, d->F, lo, head, d->tkey,
                                                                           d->tseq, d->T);
      count_launch();
    }
    d->used = head - lo;
  }
  // 2. keys, batch duplicates, hits, and the misses' seqs
  B2RL_CUDA(cudaMemsetAsync(d->bkey, 0xFF, sizeof(unsigned long long) * (size_t)d->BT, st));
  B2RL_CUDA(cudaMemsetAsync(d->bpos, 0x7F, sizeof(int32_t) * (size_t)d->BT, st));
  k_dedup_hash<L><<<warps_grid(frames), DD_THREADS, 0, st>>>(s_dev, ns_dev, frames, d->mask, d->key, d->bkey, d->bpos,
                                                          d->BT);
  const bool coded = d->P > 0;
  const ResolveArgs A{s_dev, ns_dev, frames, d->key, d->bkey, d->bpos, d->BT, d->tkey, d->tseq, d->T, d->pool, d->F,
                      head - d->W, d->rep, d->fseq, d->P, d->foff, d->usz};
  auto resolve = coded ? k_dedup_resolve<L, true> : k_dedup_resolve<L, false>;
  resolve<<<warps_grid(frames), DD_THREADS, 0, st>>>(A);
  k_dedup_scan<<<1, 1024, 0, st>>>(d->fseq, frames, head, d->misses_dev);
  count_launch(3);
  if (coded) {
    k_coded_offsets<<<1, 1024, 0, st>>>(d->fseq, d->usz, frames, head, d->units, d->P, d->uoff, d->misses_dev);
    count_launch();
  }
  B2RL_CHECK_LAUNCH();
  B2RL_CUDA(cudaMemcpyAsync(d->misses_host, d->misses_dev, (coded ? 2 : 1) * sizeof(int64_t), cudaMemcpyDeviceToHost,
                            st));
  B2RL_CUDA(cudaStreamSynchronize(st));
  const int64_t head_new = head + d->misses_host[0];
  const int64_t units_new = coded ? d->misses_host[1] : 0;
  // 3. the eviction rule: the oldest slots with F - W or more frames stored since their batch began lose their
  //    priority, in stream order before their frames can be overwritten; with a coded pool also those with
  //    P - (W + 1) 442 or more units written since (DESIGN.md §4.21)
  int64_t tail = h->head - h->size;
  if (tail < 0) tail += h->capacity;
  int64_t dead = 0;
  auto dies = [&](int64_t slot) {
    return head_new - d->ins[(size_t)slot] >= d->F - d->W ||
           (coded && units_new - d->uins[(size_t)slot] >= d->P - (d->W + 1) * FC_RAW_UNITS);
  };
  while (dead < h->size && dies((tail + dead) % h->capacity)) ++dead;
  if (dead > 0) {
    h->size -= dead;
    int rc = b2rl_tree_update_impl(h, nullptr, tail, nullptr, 0.0f, dead, st, true);
    if (rc != B2RL_OK) return rc;
  }
  // 4. pool ids, new frames, key table; then the other fields and the priorities as b2rl_replay_push does
  const CopyArgs C{s_dev, ns_dev, frames, d->key, d->rep, d->fseq, head, d->pool, d->pool_key, d->F, d->tkey, d->tseq,
                   d->T, (int32_t*)h->field[d->planes_field], h->head, h->capacity, d->R, d->P, d->uoff, d->usz,
                   d->foff, d->flen};
  auto copy = coded ? k_dedup_copy<L, true> : k_dedup_copy<L, false>;
  copy<<<warps_grid(frames), DD_THREADS, 0, st>>>(C);
  count_launch();
  B2RL_CHECK_LAUNCH();
  int rc = copy_ring_range(h, fields_src, h->head, n, st);
  if (rc != B2RL_OK) return rc;
  B2RL_CUDA(cudaMemcpyAsync(h->scratch_val, prios, (size_t)n * sizeof(float), cudaMemcpyDefault, st));
  for (int64_t i = 0; i < n; ++i) {
    const size_t slot = (size_t)((h->head + i) % h->capacity);
    d->ins[slot] = head;
    if (coded) d->uins[slot] = d->units;
  }
  rc = publish(h, h->scratch_val, n, st);
  if (rc != B2RL_OK) return rc;
  B2RL_CUDA(cudaEventRecord(d->done, st));
  d->head = head_new;
  d->used += head_new - head;
  d->units = units_new;
  return B2RL_OK;
}

extern "C" int b2rl_dedup_push(b2rl_replay* h, const uint8_t* s_dev, const uint8_t* ns_dev,
                               const void* const* fields_src, const float* prios, int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  DedupState* d = h->dedup;
  B2RL_REQUIRE(d != nullptr, "not a frame-deduplicated replay (b2rl_dedup_attach)");
  B2RL_REQUIRE(d->layout == Layout::Pairs, "a strip or rollout handle (b2rl_dedup_attach_strips, _rollouts) takes b2rl_dedup_push_strips");
  B2RL_REQUIRE(n >= 0 && n <= d->max_batch, "n out of range (0..max_batch of b2rl_dedup_info)");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(s_dev != nullptr && ns_dev != nullptr, "null argument");
  B2RL_REQUIRE((uintptr_t)s_dev % 16 == 0 && (uintptr_t)ns_dev % 16 == 0, "frame stacks must be 16-byte aligned");
  return dedup_push<Layout::Pairs>(h, s_dev, ns_dev, fields_src, prios, n, (cudaStream_t)stream);
}

extern "C" int b2rl_dedup_push_strips(b2rl_replay* h, const uint8_t* strips_dev, const void* const* fields_src,
                                      const float* prios, int64_t n, void* stream) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  DedupState* d = h->dedup;
  B2RL_REQUIRE(d != nullptr, "not a frame-deduplicated replay (b2rl_dedup_attach_strips)");
  B2RL_REQUIRE(d->layout == Layout::Strips, "an Ape-X handle (b2rl_dedup_attach) takes b2rl_dedup_push");
  B2RL_REQUIRE(n >= 0 && n <= d->max_batch, "n out of range (0..max_batch of b2rl_dedup_info)");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(strips_dev != nullptr, "null argument");
  B2RL_REQUIRE((uintptr_t)strips_dev % 16 == 0, "frame strips must be 16-byte aligned");
  return dedup_push<Layout::Strips>(h, strips_dev, nullptr, fields_src, prios, n, (cudaStream_t)stream);
}
