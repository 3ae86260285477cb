"""numpy restatement of the residual network's fused stem (csrc/stem.cu): the weight digits of b2rl_stem_pack, the
forward's exact integer sums and fp32 recombination (bit for bit what the kernel computes), the max-pool's first-maximum
tie rule, and the weight gradient's folded pool backward and digit arithmetic.  Any frame size H x W (the kernel runs
84 x 84), so the CPU tests can check it against float64 at a tiny size."""
import numpy as np

F32 = np.float32


def pack(w):
    """w fp32 (16, 4, 3, 3) -> (digits int64 (4, 16, 36), scale fp32 (16,) = s / 255): conv_1's pack arithmetic."""
    w = np.asarray(w, np.float32).reshape(w.shape[0], -1)
    m = np.abs(w).max(axis=1)
    s = np.where(m > 0, m / F32(127), F32(1)).astype(np.float32)
    x = w.astype(np.float64) / s.astype(np.float64)[:, None]
    q = np.empty((4,) + w.shape, np.int64)
    for j in range(4):
        r = np.clip(np.rint(x), -127, 127)
        q[j] = r
        x = (x - r) * 128.0
    return q, (s / F32(255)).astype(np.float32)


def patches(frames):
    """uint8 (n, 4, H, W) -> int64 (n, 36, H, W): the zero-padded 3x3 patch, element (c, ky, kx) = 9c + 3ky + kx."""
    n, C, H, W = frames.shape
    p = np.zeros((n, C, H + 2, W + 2), np.int64)
    p[:, :, 1:-1, 1:-1] = frames
    out = np.empty((n, C, 3, 3, H, W), np.int64)
    for ky in range(3):
        for kx in range(3):
            out[:, :, ky, kx] = p[:, :, ky:ky + H, kx:kx + W]
    return out.reshape(n, C * 9, H, W)


def conv(frames, w):
    """The kernel's conv output fp32 (n, 16, H, W): exact digit sums, recombined as conv1.cu's epilogue."""
    q, scale = pack(w)
    P = patches(frames)
    Q = np.einsum("dce,nehw->dnchw", q, P)                                   # exact int64 digit sums
    fu = (Q[0] * 128 + Q[1]).astype(np.float32)
    ft = (Q[2] * 128 + Q[3]).astype(np.float32)
    v = (ft.astype(np.float64) * 2.0 ** -14 + fu.astype(np.float64)).astype(np.float32)   # one fma
    sc = (scale * F32(1 / 128)).astype(np.float32)
    return (v * sc[None, :, None, None]).astype(np.float32)


def pool(y):
    """3x3 / stride-2 / pad-1 max-pool of y (n, C, H, W) -> (pooled, argmax uint8 = 3i + j of the first maximum in
    row-major window order, padded positions skipped)."""
    n, C, H, W = y.shape
    PH, PW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    best = np.full((n, C, PH, PW), -np.inf, np.float32)
    arg = np.zeros((n, C, PH, PW), np.uint8)
    for i in range(3):
        for j in range(3):
            ys, xs = 2 * np.arange(PH) - 1 + i, 2 * np.arange(PW) - 1 + j
            ok = (ys[:, None] >= 0) & (ys[:, None] < H) & (xs[None, :] >= 0) & (xs[None, :] < W)
            v = y[:, :, np.clip(ys, 0, H - 1)][:, :, :, np.clip(xs, 0, W - 1)]
            take = ok & (v > best)
            best = np.where(take, v, best)
            arg = np.where(take, np.uint8(3 * i + j), arg)
    return best, arg


def fold(gp, arg, H, W, dtype=np.float32):
    """The conv output's gradient (n, C, H, W): each position sums, in (py, px) order, the pooled gradients whose
    window chose it (at most four)."""
    n, C, PH, PW = gp.shape
    g = np.zeros((n, C, H, W), dtype)
    for y in range(H):
        pys = [y // 2] + ([y // 2 + 1] if y % 2 and y // 2 + 1 < PH else [])
        for x in range(W):
            pxs = [x // 2] + ([x // 2 + 1] if x % 2 and x // 2 + 1 < PW else [])
            s = np.zeros((n, C), dtype)
            for py in pys:
                for px in pxs:
                    hit = arg[:, :, py, px] == 3 * (y - 2 * py + 1) + (x - 2 * px + 1)
                    s = np.where(hit, (s + gp[:, :, py, px].astype(dtype)).astype(dtype), s)
            g[:, :, y, x] = s
    return g


def digit_exponent(absmax):
    t = np.asarray(absmax, np.float32) / F32(127)
    e = ((t.view(np.uint32) >> 23) & 0xFF).astype(np.int64) + 1
    return np.clip(e, 27, 227)


def wgrad(frames, gp, arg):
    """dW (16, 36) in float64 from the kernel's arithmetic per stack: folded fp32 gy, balanced base-256 digits against
    s > 4 max|gp| / 127 (a power of two), exact integer sums, scaled and divided by 255.  The kernel sums the same
    per-stack terms in a different fp64 order."""
    n, C, H, W = frames.shape[0], gp.shape[1], frames.shape[2], frames.shape[3]
    g = fold(gp, arg, H, W)
    P = patches(frames).reshape(n, 36, -1)
    e = digit_exponent(4 * np.abs(gp).reshape(n, C, -1).max(axis=2))          # (n, C)
    inv = np.ldexp(1.0, 24 - (e - 127))
    X = np.rint(g.reshape(n, C, -1).astype(np.float64) * inv[:, :, None]).astype(np.int64)   # exact: power-of-two scale
    S = np.einsum("nck,nek->nce", X, P).astype(np.float64)                    # exact integer sums
    return (S * np.ldexp(1.0, e - 127 - 24)[:, :, None]).sum(axis=0) / 255.0
