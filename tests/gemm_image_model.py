"""A NumPy statement of the 3xTF32 operand image (csrc/operand_image.cuh), of how csrc/gemm.cu splits K, and of the
GEMM that reads the images, plus operands whose 3xTF32 product is exact at every intermediate.

Host only (no torch.cuda): tests/test_gemm_image_model_cpu.py checks the model itself and shows that the emulated GEMM
changes under each layout, pipeline and split error the exact GPU test (tests/test_gpu_39_gemm_exact.py) is meant to
catch; the GPU test compares every image writer and the GEMM with this model bit for bit."""
from __future__ import annotations

import numpy as np

KC = 32                         # contraction padding and K-split unit (floats)
KH = 16                         # floats of one half-chunk: one pipeline stage, 64-byte image rows
TM, TN = 128, 256               # tile rows of the A and of the B image
STAGES = 4                      # k_gemm_tf32x3's shared-memory ring
MAX_CHUNKS_PER_SPLIT = 32       # gemm.cu: K chunks one split accumulates at most

# exact_operands: |hi*hi + hi*lo + lo*hi| of one product is below this, and the products lie on the 2^-11 grid
PRODUCT_BOUND = 9.01
MAX_NNZ = 200                   # MAX_NNZ * PRODUCT_BOUND < 2^11: every partial sum has at most 22 significant bits
LO = 2.0 ** -11


def ceil_div(a: int, b: int) -> int:
    return -(-a // b)


def tile_rows(b_role: bool) -> int:
    return TN if b_role else TM


# --------------------------------------------------------------------------------------------------------------------- #
# the split and the layout                                                                                              #
# --------------------------------------------------------------------------------------------------------------------- #
def split_tf32(x):
    """(hi, lo) of fp32 x as image::split_tf32 forms them: hi rounds the 13 dropped mantissa bits to nearest with ties
    away from zero in magnitude; where that rounding reaches inf, hi is x truncated; non-finite x gives hi = x (payload
    kept) and lo = 0; otherwise lo = x - hi, exact in fp32."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32)
    h = (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)                  # uint32 arithmetic wraps like the kernel's
    overflow = (h & np.uint32(0x7F800000)) == np.uint32(0x7F800000)
    h = np.where(overflow, u & np.uint32(0xFFFFE000), h)
    nonfinite = (u & np.uint32(0x7F800000)) == np.uint32(0x7F800000)
    hi_bits = np.where(nonfinite, u, h).astype(np.uint32)
    hi = hi_bits.view(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = np.where(nonfinite, np.float32(0.0), x - hi).astype(np.float32)
    return hi, lo


# the split's edge inputs (bits): signed zeros, subnormals, the 13-bit ties, the largest floats whose hi stays finite or
# is truncated, FLT_MAX, infinities, quiet and signalling NaNs with payloads
SPECIAL_BITS = (0x00000000, 0x80000000, 0x00000001, 0x80001FFF, 0x007FFFFF, 0x3F801000, 0xBF801000, 0x3F800FFF,
                0x3F803000, 0x7F7FEFFF, 0x7F7FF000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000,
                0x7FC01234, 0xFFFFFFFF, 0x7F800001, 0xFFA00FFF)


def rows_pad(rows: int, b_role: bool) -> int:
    tr = tile_rows(b_role)
    return ceil_div(rows, tr) * tr


def term_stride(k_chunks: int, rows_padded: int) -> int:
    """Floats between the hi and the lo image."""
    return k_chunks * rows_padded * KC


def packed_floats(rows: int, k: int, b_role: bool) -> int:
    """b2rl_gemm_packed_floats: both terms of the image."""
    return 2 * term_stride(ceil_div(k, KC), rows_pad(rows, b_role))


def offset(row, k, tile_rows_: int, rows_padded: int, xor: bool = True):
    """Float offset (in one term) of the 16-byte unit holding contraction elements k .. k + 3 (k a multiple of 4) of
    image row `row`: [k_half][row_tile][row_in_tile][16-byte unit XOR ((row_in_tile >> 1) & 3)].  Vectorised over
    row and k.  xor=False is the layout without the swizzle (a mutant of the tests)."""
    row = np.asarray(row, dtype=np.int64)
    k = np.asarray(k, dtype=np.int64)
    rt, rr = row // tile_rows_, row % tile_rows_
    kh, unit = k // KH, (k // 4) & 3
    if xor:
        unit = unit ^ ((rr >> 1) & 3)
    return ((kh * (rows_padded // tile_rows_) + rt) * tile_rows_ + rr) * KH + (unit << 2)


def _unit_offsets(n_rows_pad: int, k_chunks: int, tr: int, xor: bool = True) -> np.ndarray:
    """[rows_pad][k_chunks * 8] offsets of every 16-byte unit of one term."""
    rows = np.arange(n_rows_pad, dtype=np.int64)[:, None]
    ks = (np.arange(k_chunks * 8, dtype=np.int64) * 4)[None, :]
    return offset(rows, ks, tr, n_rows_pad, xor)


def image(mat, transpose: bool, b_role: bool) -> np.ndarray:
    """The {hi, lo} image of fp32 `mat` (or of its transpose): float32[packed_floats], every padding float zero."""
    op = np.asarray(mat, dtype=np.float32)
    if transpose:
        op = op.T
    rows, k = op.shape
    tr, rp, kc = tile_rows(b_role), rows_pad(rows, b_role), ceil_div(k, KC)
    padded = np.zeros((rp, kc * KC), dtype=np.float32)
    padded[:rows, :k] = op
    hi, lo = split_tf32(padded)
    ts = term_stride(kc, rp)
    out = np.zeros(2 * ts, dtype=np.float32)
    idx = _unit_offsets(rp, kc, tr)[:, :, None] + np.arange(4, dtype=np.int64)
    out[idx] = hi.reshape(rp, kc * 8, 4)
    out[ts + idx] = lo.reshape(rp, kc * 8, 4)
    return out


def pieces_image(mats, transpose: bool, b_role: bool) -> np.ndarray:
    """linear._pack_pieces: the image of the vertically stacked `mats` (transpose=False), or of the transpose of that
    stack, where the pieces sit side by side along the contraction index (transpose=True)."""
    return image(np.concatenate([np.asarray(m, dtype=np.float32) for m in mats], 0), transpose, b_role)


def act_flat(y_nhwc, relu: bool) -> np.ndarray:
    """x[b][f] with f = c*HW + hw of y[b][hw][c] (nn.Flatten of the NCHW tensor), after the ReLU if `relu`."""
    y = np.asarray(y_nhwc, dtype=np.float32)
    if relu:
        y = np.maximum(y, np.float32(0.0))
    B, HW, C = y.shape
    return np.ascontiguousarray(y.transpose(0, 2, 1).reshape(B, C * HW))


def act_image(y_nhwc, relu: bool, transpose: bool) -> np.ndarray:
    """b2rl_gemm_pack_act_nhwc: the A-role image of x = flatten(relu(y)) [B][C*HW] (transpose=False) or the B-role
    image of x^T [C*HW rows][B contraction] (transpose=True)."""
    x = act_flat(y_nhwc, relu)
    return image(x, transpose, transpose)


def read_image(img, rows: int, k: int, b_role: bool, xor: bool = True):
    """(hi, lo) float32 [rows_pad][k_chunks * 32] read back from an image through `offset`."""
    tr, rp, kc = tile_rows(b_role), rows_pad(rows, b_role), ceil_div(k, KC)
    ts = term_stride(kc, rp)
    img = np.asarray(img, dtype=np.float32)
    assert img.size == 2 * ts, (img.size, 2 * ts)
    idx = _unit_offsets(rp, kc, tr, xor)[:, :, None] + np.arange(4, dtype=np.int64)
    return img[idx].reshape(rp, kc * KC), img[ts + idx].reshape(rp, kc * KC)


# --------------------------------------------------------------------------------------------------------------------- #
# the K split                                                                                                           #
# --------------------------------------------------------------------------------------------------------------------- #
def splits(M: int, N: int, K: int, sms: int) -> int:
    """gemm.cu's gemm_splits: cover the SMs about once, at most MAX_CHUNKS_PER_SPLIT chunks per split, no empty
    trailing split."""
    tiles = ceil_div(M, TM) * ceil_div(N, TN)
    kc = ceil_div(K, KC)
    s = max(1, sms // max(tiles, 1))
    s = min(s, kc)
    if s * MAX_CHUNKS_PER_SPLIT < kc:
        s = ceil_div(kc, MAX_CHUNKS_PER_SPLIT)
    per = ceil_div(kc, s)
    return ceil_div(kc, per)


def split_range(K: int, n_splits: int, z: int) -> tuple[int, int]:
    """[c0, c1): the 32-float chunks split z of n_splits accumulates (k_gemm_tf32x3's k0, k1)."""
    kc = ceil_div(K, KC)
    per = ceil_div(kc, n_splits)
    c0 = z * per
    return c0, min(c0 + per, kc)


def depths(K: int, n_splits: int) -> list[int]:
    """nk of every split: the half-chunks its pipeline runs through."""
    return [2 * (c1 - c0) for c0, c1 in (split_range(K, n_splits, z) for z in range(n_splits))]


# --------------------------------------------------------------------------------------------------------------------- #
# the GEMM                                                                                                              #
# --------------------------------------------------------------------------------------------------------------------- #
MUTANTS = ("no_xor", "drop_lo_half", "stale_stage", "split_off_by_one", "add_lo_lo")


def emulate(a_img, b_img, M: int, N: int, K: int, sms: int, mutant: str | None = None, n_splits: int | None = None):
    """k_gemm_tf32x3 in float64, reading both images through `offset`: per split z the sum over its half-chunks of
    lo*hi + hi*lo + hi*hi (lo*lo dropped) -> (partials [splits][M][N], their sum in split order).

    `mutant` emulates one error the exact GPU test must catch:
      no_xor            the reader ignores the swizzle
      drop_lo_half      both lo terms of one half-chunk (the middle one of the contraction) left out
      stale_stage       the last half-chunk of every split whose pipeline wraps the ring (nk > STAGES) multiplies the
                        tiles of half-chunk nk - 1 - STAGES, still in that stage
      split_off_by_one  every split starts one half-chunk late
      add_lo_lo         the fourth product lo*lo added"""
    assert mutant is None or mutant in MUTANTS, mutant
    if n_splits is None:
        n_splits = splits(M, N, K, sms)
    xor = mutant != "no_xor"
    a_hi, a_lo = (t[:M].astype(np.float64) for t in read_image(a_img, M, K, False, xor))
    b_hi, b_lo = (t[:N].astype(np.float64) for t in read_image(b_img, N, K, True, xor))
    if mutant == "drop_lo_half":
        h = (ceil_div(K, KH) - 1) // 2
        a_lo[:, h * KH:(h + 1) * KH] = 0.0
        b_lo[:, h * KH:(h + 1) * KH] = 0.0
    parts = np.zeros((n_splits, M, N), dtype=np.float64)
    for z in range(n_splits):
        c0, c1 = split_range(K, n_splits, z)
        h0, h1 = 2 * c0, 2 * c1
        if mutant == "split_off_by_one":
            h0 += 1
        order = list(range(h0, h1))                     # the half-chunks this split's pipeline multiplies
        if mutant == "stale_stage" and len(order) > STAGES:
            order[-1] = order[-1 - STAGES]
        cols = (np.asarray(order, dtype=np.int64)[:, None] * KH + np.arange(KH)).ravel()
        ah, al, bh, bl = a_hi[:, cols], a_lo[:, cols], b_hi[:, cols], b_lo[:, cols]
        # one float64 product of the three terms: every partial here is exact (float64 has room for them all)
        parts[z] = np.concatenate([al, ah, ah], 1) @ np.concatenate([bh, bl, bh], 1).T
        if mutant == "add_lo_lo":
            parts[z] += al @ bl.T
    total = parts[0].copy()
    for z in range(1, n_splits):
        total += parts[z]
    return parts, total


def exact_product(a, b) -> np.ndarray:
    """The 3xTF32 product of fp32 A [M][K] and B [N][K] in float64: sum of a_lo*b_hi + a_hi*b_lo + a_hi*b_hi."""
    a_hi, a_lo = (t.astype(np.float64) for t in split_tf32(a))
    b_hi, b_lo = (t.astype(np.float64) for t in split_tf32(b))
    return np.concatenate([a_lo, a_hi, a_hi], 1) @ np.concatenate([b_hi, b_lo, b_hi], 1).T


# --------------------------------------------------------------------------------------------------------------------- #
# exact operands                                                                                                        #
# --------------------------------------------------------------------------------------------------------------------- #
def _values(rng, shape, nonneg: bool, lo_zero: bool = True) -> np.ndarray:
    """h + l, h in {2, 3} (signed unless nonneg), l in {0, +-2^-11} (never 0 unless lo_zero): rn_tf32 gives hi = h,
    lo = l exactly."""
    h = rng.choice(np.array([2.0, 3.0]), size=shape)
    if not nonneg:
        h = h * rng.choice(np.array([-1.0, 1.0]), size=shape)
    l_ = rng.choice(np.array([-LO, 0.0, LO]) if lo_zero else np.array([-LO, LO]), size=shape)
    return (h + l_).astype(np.float32)


def nnz_for(rows_in_tile: int, K: int, nnz: int) -> int:
    """Nonzeros per row of a row tile: `nnz`, more where the tile's rows are too few to reach every half-chunk."""
    need = ceil_div(ceil_div(K, KH), rows_in_tile)
    return min(K, max(nnz, min(MAX_NNZ, need)))


def sparse_pattern(M: int, K: int, nnz: int = 24) -> np.ndarray:
    """bool [M][K]: at most nnz_for(...) nonzeros per row, placed so that in every 128-row tile of the A image every
    half-chunk of the contraction and every (row mod 8, 16-byte unit) pair holds one, where the tile's rows can."""
    mask = np.zeros((M, K), dtype=bool)
    hc = ceil_div(K, KH)
    for t in range(ceil_div(M, TM)):
        r0 = t * TM
        rows = min(TM, M - r0)
        n = nnz_for(rows, K, nnz)
        for rr in range(rows):
            s = np.arange(n, dtype=np.int64)
            g = rr * n + s                                     # this tile's slots, consecutive over its rows
            h = g % hc                                         # ... walk the half-chunks
            u = (s + rr) % 4                                   # every row visits every 16-byte unit
            e = (s // 4 + rr // 8 + g // hc) % 4
            w = 4 * u + e
            span = np.minimum(KH, K - KH * h)                  # the last half-chunk may be short
            k = KH * h + w % span
            mask[r0 + rr, k] = True
    return mask


def coverage(mask: np.ndarray, K: int) -> list:
    """Per 128-row tile: the half-chunks and the (row mod 8, unit) pairs that hold a nonzero, and those that could."""
    M = mask.shape[0]
    hc = ceil_div(K, KH)
    out = []
    for t in range(ceil_div(M, TM)):
        sub = mask[t * TM:(t + 1) * TM]
        rr, k = np.nonzero(sub)
        halves = set((k // KH).tolist())
        pairs = set(zip((rr % 8).tolist(), ((k // 4) % 4).tolist()))
        units_real = sorted(set(((np.arange(K) // 4) % 4).tolist()))
        possible_pairs = {(c, u) for c in set((np.arange(sub.shape[0]) % 8).tolist()) for u in units_real}
        out.append({"halves": halves, "pairs": pairs, "all_halves": set(range(hc)), "all_pairs": possible_pairs,
                    "rows": sub.shape[0], "max_nnz": int(sub.sum(1).max())})
    return out


def exact_operands(M: int, N: int, K: int, seed: int, nnz: int = 24, nonneg_a: bool = False,
                   nonneg_b: bool = False):
    """(A [M][K], B [N][K]) fp32 whose 3xTF32 product is exact in fp32 at every intermediate.

    Values are h + l with h in {+-2, +-3}, l in {0, +-2^-11}, or 0: hi = h, lo = l, so every hi*hi, hi*lo and lo*hi
    lies on the 2^-11 grid and is below PRODUCT_BOUND in magnitude.  A is row-sparse (sparse_pattern), at most MAX_NNZ
    nonzeros per row, so every sum of any subset of one output's products, in any order, is below 2^11 on the 2^-11
    grid: at most 22 significant bits, exact in the tensor cores' fp32 accumulation, in every split partial and in the
    split reduction.  B is dense.  lo*lo is nonzero for many outputs, so a fourth product changes them."""
    rng = np.random.default_rng(seed)
    mask = sparse_pattern(M, K, nnz)
    per_row = mask.sum(1)
    assert per_row.max() <= MAX_NNZ and per_row.max() * PRODUCT_BOUND < 2.0 ** 11, per_row.max()
    for cov in coverage(mask, K):
        reach = min(len(cov["all_halves"]), cov["rows"] * MAX_NNZ)
        assert len(cov["halves"]) >= reach, (M, K, len(cov["halves"]), reach)
        if cov["rows"] >= 8 and cov["max_nnz"] >= 4:
            assert cov["pairs"] == cov["all_pairs"], (M, K, sorted(cov["all_pairs"] - cov["pairs"]))
    a = np.zeros((M, K), dtype=np.float32)
    a[mask] = _values(rng, int(mask.sum()), nonneg_a, lo_zero=False)     # every lo of A is nonzero
    b = _values(rng, (N, K), nonneg_b)
    return a, b


def relu_preimage(x, seed: int) -> np.ndarray:
    """y with relu(y) == x for nonnegative x: x where x > 0, a negative value of the same set elsewhere."""
    x = np.asarray(x, dtype=np.float32)
    assert (x >= 0).all()
    neg = -_values(np.random.default_rng(seed), x.shape, True)
    return np.where(x > 0, x, neg).astype(np.float32)


# --------------------------------------------------------------------------------------------------------------------- #
# the exact GPU test's GEMM grid                                                                                        #
# --------------------------------------------------------------------------------------------------------------------- #
# Pipeline depth: 1536 x 3072 is 144 output tiles, so the grid has one split on any card with at most 287 SMs, and K
# alone sets nk, the half-chunks the four-stage ring runs through (64: the 32-chunk cap of one split).
DEPTH_M, DEPTH_N = 1536, 3072
DEPTH_K = {2: 32, 4: 64, 6: 96, 8: 128, 10: 160, 16: 256, 64: 1024}

WRITER_SIZES = (1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 255, 256, 257, 3136)
EDGE_M = (1, 2, 63, 64, 65, 127, 128, 129, 257)
EDGE_N = (1, 2, 3, 5, 255, 256, 257, 511)
EDGE_K = (1, 4, 5, 31, 33, 127, 129, 255, 257, 3136)


def edge_shapes():
    """(M, N, K, ldc) at the tile edges: every M with every N, K walking EDGE_K, ldc = ceil4(N) or 8 wider."""
    out = []
    for i, M in enumerate(EDGE_M):
        for j, N in enumerate(EDGE_N):
            q = i * len(EDGE_N) + j
            K = EDGE_K[q % len(EDGE_K)]
            ldc = ceil_div(N, 4) * 4 + (8 if q % 2 else 0)
            out.append((M, N, K, ldc))
    return out
