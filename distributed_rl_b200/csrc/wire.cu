// The actors' pickled records decoded on the GPU (DESIGN.md §4.24).  wire.py derives a template from one record: run
// lists that sort every byte into skeleton (compared with the template's bytes), value spans (converted into the
// decoded batch's fields) and free spans (ignored).  b2rl_wire_decode checks n records of one template against it and
// scatters their values; b2rl_wire_gather packs the records' blobs into pinned staging without the GIL.
#include "common.cuh"

#include <math.h>

namespace b2rl {

constexpr int WIRE_THREADS = 256;
enum { RUN_SKELETON = 0, RUN_SAME = 1, RUN_COPY = 2, RUN_STRIP = 3, RUN_CONVERT = 4 };
enum { S_U8, S_U16, S_I32, S_I64, S_F32, S_F64, S_F64BE, S_BOOLOP, S_B1, S_KINDS };
enum { D_I32, D_F32, D_F32_DIRECT, D_U8_BOOL, D_F32_NOT, D_KINDS };
enum { ST_SKELETON = 1, ST_RANGE = 2, ST_NO_SLIDE = 4 };
constexpr int FRAME = 84 * 84, STACK = 4 * FRAME;

struct WireFields {
  uint8_t* ptr[B2RL_MAX_FIELDS];
  int64_t row[B2RL_MAX_FIELDS];
};

__device__ __forceinline__ uint64_t load_le(const uint8_t* p, int n) {
  uint64_t v = 0;
  for (int i = n - 1; i >= 0; --i) v = (v << 8) | p[i];
  return v;
}

// double -> float32 as the host's cast does: round to nearest even, and a NaN keeps its sign and the top of its
// payload, quieted.  The NaN case is spelled out rather than left to cvt.rn.f32.f64, although on an H100 that
// instruction returned the same bits for 2^20 random NaN payloads (so __double2float_rn alone decodes the same there).
__device__ __forceinline__ uint32_t f64_to_f32_bits(uint64_t b) {
  const double d = __longlong_as_double((long long)b);
  if (isnan(d)) return (uint32_t)(b >> 32 & 0x80000000u) | 0x7fc00000u | (uint32_t)(b >> 29 & 0x003fffffu);
  return __float_as_uint(__double2float_rn(d));
}

// One element: source kind sk at p -> destination kind dk at q.  Returns status bits.
__device__ __forceinline__ int convert(const uint8_t* p, int sk, uint8_t* q, int dk) {
  bool is_float = false;
  int64_t i = 0;
  uint64_t f = 0;        // bits of the double, or of the float32 for S_F32
  switch (sk) {
    case S_U8: i = p[0]; break;
    case S_U16: i = (int64_t)load_le(p, 2); break;
    case S_I32: i = (int32_t)(uint32_t)load_le(p, 4); break;
    case S_I64: i = (int64_t)load_le(p, 8); break;
    case S_F32: is_float = true; f = load_le(p, 4); break;
    case S_F64: is_float = true; f = load_le(p, 8); break;
    case S_F64BE: {
      is_float = true;
      for (int k = 0; k < 8; ++k) f = (f << 8) | p[k];
      break;
    }
    case S_BOOLOP:
      if (p[0] != 0x88 && p[0] != 0x89) return ST_SKELETON;    // NEWTRUE / NEWFALSE
      i = p[0] == 0x88;
      break;
    case S_B1: i = p[0] != 0; break;
    default: return ST_SKELETON;
  }
  double fv = 0.0;
  if (is_float) fv = sk == S_F32 ? (double)__uint_as_float((uint32_t)f) : __longlong_as_double((long long)f);
  const bool truth = is_float ? fv != 0.0 : i != 0;             // NaN != 0: true, as bool(nan) is
  uint32_t out = 0;
  switch (dk) {
    case D_I32:
      if (is_float) return ST_SKELETON;
      if (i < INT32_MIN || i > INT32_MAX) return ST_RANGE;
      out = (uint32_t)(int32_t)i;
      break;
    case D_F32:
    case D_F32_DIRECT:
      // float(x) widens a float32 to double, which quiets a signalling NaN; numpy's float32 array cast keeps its bits
      if (sk == S_F32) out = (uint32_t)f | (dk == D_F32 && (f & 0x7fffffffu) > 0x7f800000u ? 0x00400000u : 0u);
      else if (is_float) out = f64_to_f32_bits(f);
      else if (dk == D_F32) out = __float_as_uint(__double2float_rn(__ll2double_rn(i)));   // float(int), then float32
      else out = __float_as_uint(__ll2float_rn(i));                                        // numpy's int -> float32
      break;
    case D_U8_BOOL: *q = truth; return 0;
    case D_F32_NOT: out = __float_as_uint(truth ? 0.0f : 1.0f); break;
    default: return ST_SKELETON;
  }
  q[0] = out & 0xff; q[1] = out >> 8 & 0xff; q[2] = out >> 16 & 0xff; q[3] = out >> 24;
  return 0;
}

// 16 bytes starting m bytes into the aligned pair (lo, hi).
__device__ __forceinline__ uint4 shift16(uint4 lo, uint4 hi, int m) {
  uint32_t a0, a1, a2, a3, a4;
  switch (m >> 2) {
    case 0: a0 = lo.x; a1 = lo.y; a2 = lo.z; a3 = lo.w; a4 = hi.x; break;
    case 1: a0 = lo.y; a1 = lo.z; a2 = lo.w; a3 = hi.x; a4 = hi.y; break;
    case 2: a0 = lo.z; a1 = lo.w; a2 = hi.x; a3 = hi.y; a4 = hi.z; break;
    default: a0 = lo.w; a1 = hi.x; a2 = hi.y; a3 = hi.z; a4 = hi.w; break;
  }
  const int s = (m & 3) * 8;
  return make_uint4(__funnelshift_r(a0, a1, s), __funnelshift_r(a1, a2, s), __funnelshift_r(a2, a3, s),
                    __funnelshift_r(a3, a4, s));
}

// dst[0, n) = src[0, n) by the CTA: 16-byte stores to an aligned dst, each built from two aligned 16-byte loads of the
// source (the staging keeps 16 readable bytes after every blob).
__device__ void copy_bytes(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, int64_t n) {
  int64_t done = 0;
  if (((uintptr_t)dst & 15) == 0) {
    const int m = (int)((uintptr_t)src & 15);
    const uint4* a = reinterpret_cast<const uint4*>(src - m);
    uint4* d = reinterpret_cast<uint4*>(dst);
    const int64_t nv = n >> 4;
    if (m == 0) {
      for (int64_t v = threadIdx.x; v < nv; v += blockDim.x) d[v] = __ldcs(a + v);
    } else {
      for (int64_t v = threadIdx.x; v < nv; v += blockDim.x) d[v] = shift16(__ldcs(a + v), __ldcs(a + v + 1), m);
    }
    done = nv << 4;
  }
  for (int64_t b = done + threadIdx.x; b < n; b += blockDim.x) dst[b] = src[b];
}

__device__ int differs(const uint8_t* a, const uint8_t* b, int64_t n) {
  int bad = 0;
  for (int64_t k = threadIdx.x; k < n; k += blockDim.x) bad |= a[k] != b[k];
  return bad;
}

// grid (records, tasks): CTA (r, k) runs runs[tasks[2k], tasks[2k + 1]) on record r of the staged blobs, writing its
// values to row rows[r] (r when rows is null) of each field and OR-ing what it found into status[row].
__global__ void __launch_bounds__(WIRE_THREADS)
k_wire_decode(const uint8_t* __restrict__ blobs, int64_t stride, const int32_t* __restrict__ lengths, int64_t n,
              const uint8_t* __restrict__ tmpl, int32_t tmpl_len, const int32_t* __restrict__ runs,
              const int32_t* __restrict__ tasks, const int32_t* __restrict__ rows, const __grid_constant__ WireFields out,
              int32_t* __restrict__ status) {
  __shared__ int bad_any;
  const int64_t r = blockIdx.x;
  const int64_t row = rows ? rows[r] : r;
  if (threadIdx.x == 0) bad_any = 0;
  __syncthreads();
  int bad = 0;
  if (lengths[r] != tmpl_len) {
    bad = ST_SKELETON;             // a truncated or longer blob: its bytes are not read at all
  } else {
    const uint8_t* rec = blobs + r * stride;
    for (int j = tasks[2 * blockIdx.y]; j < tasks[2 * blockIdx.y + 1]; ++j) {
      const int32_t* run = runs + 8 * j;
      const int op = run[0], src = run[1], len = run[2], field = run[3], dst = run[4], count = run[5], aux = run[6];
      uint8_t* q = out.ptr[field] + row * out.row[field] + dst;
      switch (op) {
        case RUN_SKELETON: bad |= differs(rec + src, tmpl + src, len) ? ST_SKELETON : 0; break;
        case RUN_SAME: bad |= differs(rec + src, rec + aux, len) ? ST_SKELETON : 0; break;
        case RUN_COPY: copy_bytes(q, rec + src, len); break;
        case RUN_STRIP:
          // stack t (= count) into frames t .. t + 3 of the strip: all four for t = 0, frame 3 after that; then
          // frames 1..3 of stack t must be frames 0..2 of stack t + 1 (replay.encode_strip)
          if (count == 0) copy_bytes(q, rec + src, STACK);
          else copy_bytes(q + (int64_t)(count + 3) * FRAME, rec + src + 3 * FRAME, FRAME);
          if (aux >= 0) bad |= differs(rec + src + FRAME, rec + aux, 3 * FRAME) ? ST_NO_SLIDE : 0;
          break;
        case RUN_CONVERT: {
          const int sk = run[7] & 0xff, dk = run[7] >> 8;
          const int sb = len / count, db = dk == D_U8_BOOL ? 1 : 4;
          for (int e = threadIdx.x; e < count; e += blockDim.x) bad |= convert(rec + src + e * sb, sk, q + e * db, dk);
          break;
        }
        default: bad |= ST_SKELETON;
      }
    }
  }
  if (bad) atomicOr(&bad_any, bad);
  __syncthreads();
  if (threadIdx.x == 0 && bad_any) atomicOr(status + row, bad_any);
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_wire_decode(const uint8_t* blobs_dev, int64_t stride, const int32_t* lengths_dev, int64_t n,
                                const uint8_t* tmpl_dev, int32_t tmpl_len, const int32_t* runs_dev, int32_t n_runs,
                                const int32_t* tasks_dev, int32_t n_tasks, const int32_t* rows_dev,
                                void* const* fields_dev, const int64_t* row_bytes, int32_t n_fields,
                                int32_t* status_dev, int64_t n_rows, void* stream) {
  B2RL_REQUIRE(n >= 0 && n <= INT32_MAX, "n must be in [0, 2^31)");
  B2RL_REQUIRE(n_fields >= 1 && n_fields <= B2RL_MAX_FIELDS, "n_fields must be in [1, B2RL_MAX_FIELDS]");
  B2RL_REQUIRE(fields_dev != nullptr && row_bytes != nullptr, "fields_dev and row_bytes are host arrays of n_fields");
  B2RL_REQUIRE(tmpl_len > 0 && stride >= (int64_t)tmpl_len + 16 && stride % 16 == 0,
               "stride must be a multiple of 16 with 16 readable bytes after a template-length blob");
  B2RL_REQUIRE(n_runs > 0 && n_tasks > 0 && n_tasks <= 65535, "a template has runs and 1 .. 65535 tasks");
  B2RL_REQUIRE(n_rows >= n, "n_rows (rows of the fields and of status) must be at least n");
  WireFields f{};
  for (int i = 0; i < n_fields; ++i) {
    B2RL_REQUIRE(fields_dev[i] != nullptr && row_bytes[i] > 0, "every field needs a pointer and a row size");
    f.ptr[i] = (uint8_t*)fields_dev[i];
    f.row[i] = row_bytes[i];
  }
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(blobs_dev && lengths_dev && tmpl_dev && runs_dev && tasks_dev && status_dev,
               "blobs, lengths, template, runs, tasks and status must be device pointers");
  B2RL_REQUIRE((uintptr_t)blobs_dev % 16 == 0, "the staged blobs must be 16-byte aligned");
  const dim3 grid((unsigned)n, (unsigned)n_tasks);
  k_wire_decode<<<grid, WIRE_THREADS, 0, (cudaStream_t)stream>>>(blobs_dev, stride, lengths_dev, n, tmpl_dev, tmpl_len,
                                                                 runs_dev, tasks_dev, rows_dev, f, status_dev);
  count_launch();
  B2RL_CHECK_LAUNCH();
  return B2RL_OK;
}

extern "C" int b2rl_wire_gather(const void* const* src, const int64_t* lengths, int64_t n, uint8_t* dst,
                                int64_t stride, int32_t* lengths_out) {
  B2RL_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return B2RL_OK;
  B2RL_REQUIRE(src && lengths && dst && lengths_out, "src, lengths, dst and lengths_out must be non-null");
  for (int64_t i = 0; i < n; ++i) {
    B2RL_REQUIRE(src[i] != nullptr && lengths[i] >= 0 && lengths[i] <= stride, "a blob is null or longer than stride");
  }
  for (int64_t i = 0; i < n; ++i) {
    memcpy(dst + i * stride, src[i], (size_t)lengths[i]);
    lengths_out[i] = (int32_t)lengths[i];
  }
  return B2RL_OK;
}
