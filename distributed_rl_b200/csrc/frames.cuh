// Where a frame row lives: the frame source of conv_1's forward (conv1.cu) and weight-gradient (conv1_wgrad.cu)
// kernels, and the plane address of the frame-deduplicated store's row copies (bulk_rows.cuh).
//
// A row is one 28 224-byte frame stack (four 84x84 uint8 frames).  The host turns a b2rl_frames descriptor
// (include/b2rl.h) into a FrameSource and its FrameKind once; the kernels take the kind as a template parameter, so
// each kind is its own instantiation with only its own address arithmetic.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "frame_codec.cuh"
#include "hopper.cuh"

namespace b2rl {

constexpr int PLANE_BYTES = 84 * 84;          // one frame: a channel of a stack, or one frame of a frame pool
constexpr int STACK_BYTES = 4 * PLANE_BYTES;  // one row

enum class FrameKind {
  Direct,   // row r at base + r * row_stride
  Table,    // the same, with the base read from a device-resident entry when the kernel starts
  Planes,   // channel c of row r is pool frame planes[plane_stride r + plane_base + c]
  CodedPlanes,   // the same ids at stride 8, each naming an encoding in a coded pool's unit ring (frame_codec.cuh),
                 // decoded on chip by the kernel's decoding warps instead of copied (decode_frame)
};

struct FrameSource {
  const uint8_t* base;           // Direct: the first row; Planes: the frame pool
  const uint8_t* const* table;   // Table: the entry that holds the first row's address
  const int32_t* planes;         // Planes: pool ids, plane_stride per row
  int64_t row_stride;            // Direct, Table: bytes between rows
  int64_t table_off;             // Table: bytes added to the entry's address (the rows of earlier split launches)
  int64_t rows;                  // indices are clamped to [0, rows)
  int32_t plane_base;            // Planes: 0 or 4 at stride 8, 0 at strides 1 and 4
  int32_t plane_stride;          // Planes: 8 (Ape-X s / s'), 1 (the windows of R2D2 strip records) or 4 (the stacks
                                 // of IMPALA rollout records)
  const int64_t* foff;           // CodedPlanes: absolute unit offset of each of the pool's entries
  int64_t units, entries;        // CodedPlanes: P (units in the ring) and F (entries)
};

// Frame c of plane-table row `row`: pool ids are `stride` apart from row to row.
__device__ __forceinline__ const uint8_t* plane_ptr(const uint8_t* pool, const int32_t* planes, int64_t row,
                                                    int32_t stride, int32_t plane_base, int c) {
  return pool + (int64_t)planes[row * stride + plane_base + c] * PLANE_BYTES;
}

// The address rows are read from: the base (the pool for Planes), or the table entry's as the kernel starts.
template <FrameKind KIND>
__device__ __forceinline__ const uint8_t* frame_base(const FrameSource& S) {
  if constexpr (KIND == FrameKind::Table) return *S.table + S.table_off;
  return S.base;
}

// Row `row` -> `dst` in SMEM, completing STACK_BYTES of transactions on `bar`: one bulk copy of a frame stack, or
// four of a plane table's frames.  `frames` is frame_base<KIND>(S).  Never for CodedPlanes (decode_frame).
template <FrameKind KIND>
__device__ __forceinline__ void load_row(const FrameSource& S, const uint8_t* frames, int64_t row, uint8_t* dst,
                                         uint64_t* bar) {
  sm90::mbar_expect_tx(bar, STACK_BYTES);
  if constexpr (KIND == FrameKind::Planes) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
      sm90::bulk_g2s(dst + c * PLANE_BYTES, plane_ptr(frames, S.planes, row, S.plane_stride, S.plane_base, c), PLANE_BYTES, bar);
  } else {
    sm90::bulk_g2s(dst, frames + row * S.row_stride, STACK_BYTES, bar);
  }
}

// CodedPlanes: the encoding of frame c of row `row`, at fc_entry's address for its id.
__device__ __forceinline__ const uint8_t* coded_frame(const FrameSource& S, int64_t row, int c) {
  return fc_entry(S.base, S.units, S.foff, S.entries, S.planes[row * S.plane_stride + S.plane_base + c]);
}

// NWARPS warps decode the encoding e into the frame dst (16-byte aligned, shared memory) together, as barrier `bar`;
// this is warp wi of them.  Warp 0 prepares the row tables in rows[parity] (fc_prepare), the barrier publishes them,
// and the warps split the frame's words.  Callers alternate the parity from frame to frame: warp 0 rewrites a table
// only after the next frame's barrier, which every warp reaches once it is done reading that table.
constexpr int DECODE_TABLES = 2;
template <int NWARPS>
__device__ __forceinline__ void decode_frame(const uint8_t* e, uint8_t* dst, FcRows* rows, int parity, int bar,
                                             int wi, int lane) {
  FcRows& S = rows[parity];
  const bool rowrun = e[0] == FC_ROWRUN;   // fc_prepare's rule: any other kind reads as raw
  if (wi == 0 && rowrun) fc_prepare(e, S, lane);
  sm90::named_sync(bar, 32 * NWARPS);
  const int t = wi * 32 + lane;
  if (!rowrun) {
    const uint4* s = reinterpret_cast<const uint4*>(e + FC_HEADER);
    uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll 1
    for (int i = t; i < FC_FRAME / 16; i += 32 * NWARPS) d[i] = s[i];
  } else {
    uint32_t* d = reinterpret_cast<uint32_t*>(dst);
#pragma unroll 1
    for (int w = t; w < FC_WORDS; w += 32 * NWARPS) d[w] = fc_word(e, S, w);
  }
}

// Host: refuse a descriptor that does not name exactly one well-formed source, else fill `src` and `kind`.
inline int check_frames(const b2rl_frames* f, FrameSource& src, FrameKind& kind) {
  B2RL_REQUIRE(f != nullptr, "null b2rl_frames");
  const bool pooled = f->pool != nullptr || f->planes != nullptr || f->offsets != nullptr;
  const int sources = (f->base != nullptr) + (f->table != nullptr) + pooled;
  B2RL_REQUIRE(sources > 0, "null frame source: set exactly one of frames, frame table and frame pool");
  B2RL_REQUIRE(sources == 1, "exactly one of frames, frame table and frame pool may be set");
  B2RL_REQUIRE(f->rows >= 1, "rows must be positive");
  src = FrameSource{};
  src.rows = f->rows;
  if (pooled) {
    B2RL_REQUIRE(f->pool != nullptr && f->planes != nullptr, "null frame pool or plane table");
    B2RL_REQUIRE((uintptr_t)f->pool % 16 == 0 && (uintptr_t)f->planes % 4 == 0,
                 "the frame pool must be 16-byte aligned, the plane table 4-byte aligned");
    const int32_t stride = f->plane_stride == 0 ? 8 : f->plane_stride;
    if (f->offsets != nullptr) {   // a coded Ape-X pool (b2rl_dedup_attach_coded)
      B2RL_REQUIRE(stride == 8, "a coded frame pool is read at plane_stride 0 or 8 (Ape-X s / s') only");
      B2RL_REQUIRE(f->plane_base == 0 || f->plane_base == 4, "plane_base must be 0 or 4");
      B2RL_REQUIRE(f->pool_units > 0 && f->pool_frames > 0, "a coded frame pool needs positive pool_units and pool_frames");
      B2RL_REQUIRE(f->pool_frames < (1LL << 31), "pool_frames must be below 2^31");
      B2RL_REQUIRE((uintptr_t)f->offsets % 8 == 0, "the descriptor table must be 8-byte aligned");
      kind = FrameKind::CodedPlanes;
      src.base = f->pool, src.planes = f->planes, src.plane_base = f->plane_base, src.plane_stride = 8;
      src.foff = f->offsets, src.units = f->pool_units, src.entries = f->pool_frames;
      return B2RL_OK;
    }
    B2RL_REQUIRE(stride == 8 || stride == 1 || stride == 4,
                 "plane_stride must be 0 or 8 (Ape-X s / s'), 1 (strip windows) or 4 (rollout stacks)");
    if (stride == 8) B2RL_REQUIRE(f->plane_base == 0 || f->plane_base == 4, "plane_base must be 0 or 4");
    else B2RL_REQUIRE(f->plane_base == 0, "plane_base must be 0 at plane_stride 1 or 4");
    kind = FrameKind::Planes;
    src.base = f->pool, src.planes = f->planes, src.plane_base = f->plane_base, src.plane_stride = stride;
    return B2RL_OK;
  }
  B2RL_REQUIRE(f->row_stride > 0 && f->row_stride % 16 == 0, "the row stride must be a positive multiple of 16 bytes");
  B2RL_REQUIRE(f->base ? (uintptr_t)f->base % 16 == 0 : (uintptr_t)f->table % 8 == 0,
               "frames must be 16-byte aligned, a frame table entry 8-byte aligned");
  kind = f->base ? FrameKind::Direct : FrameKind::Table;
  src.base = f->base, src.table = f->table, src.row_stride = f->row_stride;
  return B2RL_OK;
}

// Host: the rows [off, rows) of `S` as rows [0, rows - off), for the launches a weight gradient splits n into.
inline FrameSource advance(FrameSource S, FrameKind kind, int64_t off) {
  if (kind == FrameKind::Direct) S.base += off * S.row_stride;
  else if (kind == FrameKind::Table) S.table_off += off * S.row_stride;
  else S.planes += S.plane_stride * off;
  S.rows -= off;
  return S;
}

// Host: f(std::integral_constant<FrameKind, kind>{}), so that a launch site names each kernel's kind once.
template <class F>
inline cudaError_t with_frame_kind(FrameKind kind, F&& f) {
  switch (kind) {
    case FrameKind::Table: return f(std::integral_constant<FrameKind, FrameKind::Table>{});
    case FrameKind::Planes: return f(std::integral_constant<FrameKind, FrameKind::Planes>{});
    case FrameKind::CodedPlanes: return f(std::integral_constant<FrameKind, FrameKind::CodedPlanes>{});
    default: return f(std::integral_constant<FrameKind, FrameKind::Direct>{});
  }
}

}  // namespace b2rl
