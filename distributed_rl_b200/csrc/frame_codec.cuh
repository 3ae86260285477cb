// The lossless per-frame codec of a compressed R2D2 frame pool (b2rl_dedup_attach_strips_coded, DESIGN.md §4.21),
// shared by the pool's ingest and its readers (dedup.cu).  One 84 x 84 uint8 frame becomes a whole number of 16-byte
// units, with no reference to any other frame, and always the same bytes:
//
//   header (16 B)  byte 0: kind (FC_RAW or FC_ROWRUN); bytes 1-2: length in units (little-endian); bytes 3-13: the
//                  84-bit row-repeat mask (bit r, at byte 3 + r / 8 bit r % 8: row r equals row r - 1; row 0 is always
//                  coded); bytes 14-15 zero
//   FC_RAW         the 7 056 pixels follow: 442 units
//   FC_ROWRUN      per coded row (in row order) its 84-bit change mask in 11 bytes (bit x: pixel x differs from pixel
//                  x - 1; bit 0 always set), then the literals (the pixels whose bit is set) of the coded rows in
//                  order, then zero bytes up to the unit boundary
//
// The row-run form is used when it is shorter than 442 units, so no frame takes more than 442 units (7 072 bytes).
// Decoding has no serial chain: pixel (r, x) of a row-run frame is the literal base(s) + popcount(mask_s bits 0..x) - 1,
// s being the last coded row <= r and base(s) a warp scan of the coded rows' popcounts.
#pragma once

#include <stdint.h>

namespace b2rl {

constexpr int FC_SIDE = 84;
constexpr int FC_FRAME = FC_SIDE * FC_SIDE;              // 7 056 bytes
constexpr int FC_HEADER = 16;
constexpr int FC_MASK = 11;                              // bytes of an 84-bit mask
constexpr int FC_RAW_UNITS = (FC_HEADER + FC_FRAME) / 16; // 442: the largest encoding
constexpr int FC_RAW_BYTES = FC_RAW_UNITS * 16;          // 7 072
constexpr int FC_WORDS = FC_FRAME / 4;                   // 1 764 words of four pixels, 21 per row
constexpr uint8_t FC_RAW = 0, FC_ROWRUN = 1;

// Per-warp scratch of fc_prepare: per coded row its change mask and the byte offset of its first literal, per row the
// coded row it repeats.
struct FcRows {
  unsigned long long lo[FC_SIDE];   // mask bits 0..63
  unsigned int hi[FC_SIDE];         // mask bits 64..83
  uint16_t base[FC_SIDE];
  uint8_t k[FC_SIDE];
};

__device__ __forceinline__ unsigned long long fc_bits_through(int x) { return ~0ULL >> (63 - x); }   // bits 0..x

// Bytes b .. b + n - 1 (n <= 8) of p, little-endian.
__device__ __forceinline__ unsigned long long fc_load_le(const uint8_t* p, int n) {
  unsigned long long v = 0;
  for (int i = 0; i < n; ++i) v |= (unsigned long long)p[i] << (8 * i);
  return v;
}

// One warp encodes one frame (16-byte aligned) into dst (16-byte aligned, room for the returned units; nullptr: size
// only).  Every lane returns the encoding's length in units.  Row r is read as three coalesced 32-pixel loads; the
// change and repeat bits come from ballots, so the two passes (size, then write) read the frame twice and keep no
// per-row state.
__device__ __forceinline__ int fc_encode(const uint8_t* __restrict__ f, uint8_t* __restrict__ dst, int lane) {
  unsigned long long rlo = 0, rhi = 0;     // the row-repeat mask
  int coded = 0, lits = 0;
  for (int pass = 0; pass < 2; ++pass) {
    int units = FC_RAW_UNITS, lit0 = 0, C = 0, L = 0;
    if (pass == 1) {
      const int bytes = FC_HEADER + FC_MASK * coded + lits;
      units = (bytes + 15) / 16;
      if (dst == nullptr) return units < FC_RAW_UNITS ? units : FC_RAW_UNITS;
      if (units >= FC_RAW_UNITS) {               // raw: the header, then the pixels as 16-byte units
        const uint4* s = reinterpret_cast<const uint4*>(f);
        uint4* d = reinterpret_cast<uint4*>(dst + FC_HEADER);
        for (int i = lane; i < FC_FRAME / 16; i += 32) d[i] = s[i];
        if (lane == 0)
          *reinterpret_cast<uint4*>(dst) = make_uint4((unsigned)FC_RAW | ((unsigned)FC_RAW_UNITS << 8), 0u, 0u, 0u);
        return FC_RAW_UNITS;
      }
      lit0 = FC_HEADER + FC_MASK * coded;
      for (int b = bytes + lane; b < 16 * units; b += 32) dst[b] = 0;   // the tail of the last unit
      if (lane < 16) {                           // the header
        uint8_t v = 0;
        if (lane == 0) v = FC_ROWRUN;
        else if (lane == 1) v = (uint8_t)(units & 0xFF);
        else if (lane == 2) v = (uint8_t)(units >> 8);
        else if (lane < 14) {
          const int b = lane - 3;
          v = (uint8_t)(b < 8 ? rlo >> (8 * b) : rhi >> (8 * (b - 8)));
        }
        dst[lane] = v;
      }
    }
    for (int r = 0; r < FC_SIDE; ++r) {
      const uint8_t* row = f + r * FC_SIDE;
      bool same = true;
      unsigned ch[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int x = lane + 32 * c;
        bool d = false;
        if (x < FC_SIDE) {
          const uint8_t v = row[x];
          d = x == 0 || v != row[x - 1];
          if (r > 0) same = same && v == row[x - FC_SIDE];
        }
        ch[c] = __ballot_sync(0xffffffffu, d);
      }
      const bool rep = r > 0 && __all_sync(0xffffffffu, same);
      if (pass == 0) {
        if (rep) {
          if (r < 64) rlo |= 1ULL << r;
          else rhi |= 1ULL << (r - 64);
        } else {
          ++coded;
          lits += __popc(ch[0]) + __popc(ch[1]) + __popc(ch[2]);
        }
        continue;
      }
      if (rep) continue;
      uint8_t* m = dst + FC_HEADER + FC_MASK * C;
      if (lane < FC_MASK) m[lane] = (uint8_t)((lane < 4 ? ch[0] >> (8 * lane)
                                               : lane < 8 ? ch[1] >> (8 * (lane - 4)) : ch[2] >> (8 * (lane - 8))));
      int before = 0;                            // literals of this row left of the 32-pixel chunk
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int x = lane + 32 * c;
        if (ch[c] >> lane & 1u)
          dst[lit0 + L + before + __popc(ch[c] & ((1u << lane) - 1u))] = row[x];
        before += __popc(ch[c]);
      }
      ++C;
      L += before;
    }
    if (pass == 1) return units;
  }
  return FC_RAW_UNITS;   // not reached
}

// One warp: the row tables of the row-run encoding e in S (a raw encoding needs none).  Returns the kind; S is ready
// for every lane when it returns.
// Any 7 072 bytes at e decode without a read outside them or outside S, whether or not an encoder wrote them (a dead
// slot's descriptor can point into newer encodings): a kind other than FC_ROWRUN is read as raw; row 0 is coded
// whatever its repeat bit says, so every row's coded row k is in [0, C) and names a mask loaded below; and the masks
// (16 + 11 C <= 940 bytes) and every literal index (kept in [0, 7 072), fc_word) stay inside the 7 072 bytes.
__device__ __forceinline__ int fc_prepare(const uint8_t* __restrict__ e, FcRows& S, int lane) {
  const int kind = e[0];
  if (kind != FC_ROWRUN) return FC_RAW;
  const unsigned long long rlo = fc_load_le(e + 3, 8) & ~1ULL, rhi = fc_load_le(e + 11, 3) & 0xFFFFFull;
  const int C = FC_SIDE - __popcll(rlo) - __popcll(rhi);
  int carry = FC_HEADER + FC_MASK * C;           // the first literal
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int k = lane + 32 * c;
    int cnt = 0;
    if (k < C) {
      const uint8_t* m = e + FC_HEADER + FC_MASK * k;
      const unsigned long long lo = fc_load_le(m, 8), hi = fc_load_le(m + 8, 3) & 0xFFFFFull;
      S.lo[k] = lo;
      S.hi[k] = (unsigned)hi;
      cnt = __popcll(lo) + __popcll(hi);
    }
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (k < C) S.base[k] = (uint16_t)(carry + incl - cnt);
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int r = lane + 32 * c;
    if (r < FC_SIDE) {
      const int reps = r < 64 ? __popcll(rlo & fc_bits_through(r))
                              : __popcll(rlo) + __popcll(rhi & fc_bits_through(r - 64));
      S.k[r] = (uint8_t)(r - reps);
    }
  }
  __syncwarp();
  return FC_ROWRUN;
}

// Word w (pixels 4w .. 4w + 3, little-endian) of a prepared row-run encoding.  A literal index is at least
// 16 + 11 C - 1 and is kept below 7 072, so the read stays inside the 7 072 bytes at e for any bytes there.
__device__ __forceinline__ uint32_t fc_word(const uint8_t* __restrict__ e, const FcRows& S, int w) {
  const int r = w / 21, x0 = 4 * (w - 21 * r);
  const int k = S.k[r];
  const unsigned long long lo = S.lo[k], hi = S.hi[k];
  const int base = S.base[k] - 1;
  uint32_t v = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int x = x0 + i;
    const int c = x < 64 ? __popcll(lo & fc_bits_through(x)) : __popcll(lo) + __popcll(hi & fc_bits_through(x - 64));
    const int b = base + c;
    v |= (uint32_t)e[b < FC_RAW_BYTES ? b : FC_RAW_BYTES - 1] << (8 * i);
  }
  return v;
}

// One warp decodes the encoding e into the frame dst (16-byte aligned).
__device__ __forceinline__ void fc_decode(const uint8_t* __restrict__ e, uint8_t* __restrict__ dst, FcRows& S,
                                          int lane) {
  if (fc_prepare(e, S, lane) == FC_RAW) {
    const uint4* s = reinterpret_cast<const uint4*>(e + FC_HEADER);
    uint4* d = reinterpret_cast<uint4*>(dst);
    for (int i = lane; i < FC_FRAME / 16; i += 32) d[i] = s[i];
  } else {
    uint32_t* d = reinterpret_cast<uint32_t*>(dst);
    for (int w = lane; w < FC_WORDS; w += 32) d[w] = fc_word(e, S, w);
  }
  __syncwarp();     // S is free for the warp's next frame
}

// The encoding of pool id `id` in a coded pool: a ring `pool` of P 16-byte units whose entry e starts at unit
// foff[e] % P.  Any int32 names an entry (read as unsigned, % F; the attach keeps F below 2^31) and any offset a unit
// of the ring, so whatever a plane table holds the decode reads inside the pool's allocation (P units plus
// FC_RAW_BYTES: fc_prepare).  Every reader of a coded pool takes its address from here (dedup.cu's ingest and
// decoders, conv_1's coded_frame in frames.cuh), so all of them read the same bytes for the same id.
__device__ __forceinline__ const uint8_t* fc_entry(const uint8_t* pool, int64_t P, const int64_t* foff, int64_t F,
                                                   int32_t id) {
  return pool + (foff[(uint32_t)id % (uint32_t)F] % P) * 16;
}

// One warp: whether the encoding e decodes to the frame f (16-byte aligned); the same answer in every lane.
__device__ __forceinline__ bool fc_equal(const uint8_t* __restrict__ e, const uint8_t* __restrict__ f, FcRows& S,
                                         int lane) {
  bool eq = true;
  if (fc_prepare(e, S, lane) == FC_RAW) {
    const uint4* x = reinterpret_cast<const uint4*>(e + FC_HEADER);
    const uint4* y = reinterpret_cast<const uint4*>(f);
    for (int i = lane; i < FC_FRAME / 16; i += 32) {
      const uint4 u = x[i], v = y[i];
      eq = eq && u.x == v.x && u.y == v.y && u.z == v.z && u.w == v.w;
    }
  } else {
    const uint32_t* y = reinterpret_cast<const uint32_t*>(f);
    for (int w = lane; w < FC_WORDS; w += 32) eq = eq && fc_word(e, S, w) == y[w];
  }
  __syncwarp();
  return __all_sync(0xffffffffu, eq);
}

}  // namespace b2rl
