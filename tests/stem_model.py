"""numpy restatement of the residual network's fused stem (csrc/stem.cu): the weight digits of b2rl_stem_pack, the
forward's exact integer sums and fp32 recombination (bit for bit what the kernel computes), the max-pool's first-maximum
tie rule, and the weight gradient's folded pool backward and digit arithmetic.  Any frame size H x W (the kernel runs
84 x 84), so the CPU tests can check it against float64 at a tiny size.

The torch functions at the end (forward_t, wgrad_t) compute the same bits on any device, a chunk of stacks at a time,
so the GPU tests can hold the kernels to them at the learner's 21 504 stacks."""
import numpy as np
import torch

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


# --------------------------------------------------------------------------- #
# the same arithmetic in torch, on any device                                  #
# --------------------------------------------------------------------------- #
CHUNK = 256                     # frame stacks per chunk (84 x 84: 0.5 GB of float64 patches, 0.9 GB of digit sums)
WINDOWS = ((0, 0), (0, 1), (1, 0), (1, 1))      # the fold's (py, px) order: (py0, px0), (py0, px0 + 1), ...


def pow2(k):
    """2.0 ** k in float64 for an integer tensor k in [-1022, 1023], built from its exponent bits (exact)."""
    return ((k.long() + 1023) << 52).view(torch.float64)


def _rows(frames, idx, a, b):
    return frames[a:b] if idx is None else frames[idx[a:b]]


def patches_t(x):
    """uint8 (n, 4, H, W) -> float64 (n, 36, H * W): the zero-padded 3x3 patch, element (c, ky, kx) = 9c + 3ky + kx."""
    n, C, H, W = x.shape
    p = torch.nn.functional.pad(x.double(), (1, 1, 1, 1))
    out = torch.stack([p[:, :, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], 2)
    return out.reshape(n, C * 9, H * W)


def conv_t(x, w):
    """The kernel's conv output fp32 (n, 16, H, W) of uint8 stacks x: the digit sums in float64 (every partial sum an
    integer below 2^53, so exact in any order), recombined as the kernel's epilogue: fu, ft, one FMA, the scale."""
    n, _, H, W = x.shape
    q, scale = pack(w.detach().cpu().numpy())
    qd = torch.from_numpy(q.reshape(-1, 36)).to(x.device, torch.float64)        # row d * 16 + co
    Q = torch.matmul(qd, patches_t(x)).view(n, 4, -1, H, W)                    # exact integer digit sums
    fu = (Q[:, 0] * 128 + Q[:, 1]).float()
    ft = (Q[:, 2] * 128 + Q[:, 3]).float()
    v = (ft.double() * 2.0 ** -14 + fu.double()).float()                       # one fma: exact in float64, one rounding
    sc = torch.from_numpy(scale).to(x.device) * (1 / 128)                     # exact
    return v * sc.view(1, -1, 1, 1)


def pool_t(y):
    """3x3 / stride-2 / pad-1 max-pool of y (n, C, H, W) -> (pooled, argmax uint8): the first maximum in row-major
    window order (torch.argmax returns the first), padded positions skipped (-inf never wins over a finite value)."""
    n, C, H, W = y.shape
    yp = torch.nn.functional.pad(y, (1, 1, 1, 1), value=-float("inf"))
    win = yp.unfold(2, 3, 2).unfold(3, 3, 2)
    win = win.reshape(n, C, win.shape[2], win.shape[3], 9)
    a = win.argmax(-1)
    return win.gather(-1, a[..., None])[..., 0], a.to(torch.uint8)


def forward_t(frames, idx, w, chunk=CHUNK):
    """The stem forward of rows `idx` (None: all) of uint8 frames (N, 4, H, W) -> (pooled fp32, argmax uint8), bit for
    bit the kernel's, on frames' device."""
    n = frames.shape[0] if idx is None else idx.numel()
    H, W = frames.shape[-2:]
    PH, PW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    pooled = torch.empty(n, w.shape[0], PH, PW, dtype=torch.float32, device=frames.device)
    amax = torch.empty(n, w.shape[0], PH, PW, dtype=torch.uint8, device=frames.device)
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        pooled[a:b], amax[a:b] = pool_t(conv_t(_rows(frames, idx, a, b), w))
    return pooled, amax


def fold_t(gp, arg, H, W, dtype=torch.float32):
    """fold() in torch: position (y, x) sums, in `dtype` and the kernel's (py, px) order, the pooled gradients whose
    window chose it.  A window that did not choose it adds +0, which leaves the sum's bits alone."""
    n, C, PH, PW = gp.shape
    dev = gp.device
    ys, xs = torch.arange(H, device=dev), torch.arange(W, device=dev)
    a, g = arg.long(), gp.to(dtype)
    out = torch.zeros(n, C, H, W, dtype=dtype, device=dev)
    for da, db in WINDOWS:
        py, i = ys // 2 + da, ys % 2 + 1 - 2 * da                 # window row and the position's row in it
        px, j = xs // 2 + db, xs % 2 + 1 - 2 * db
        ok = ((i >= 0) & (py < PH)).view(H, 1) & ((j >= 0) & (px < PW)).view(1, W)
        pyc, pxc = py.clamp(max=PH - 1), px.clamp(max=PW - 1)
        hit = ok & (a[:, :, pyc][:, :, :, pxc] == (3 * i).view(H, 1) + j.view(1, W))
        out = out + torch.where(hit, g[:, :, pyc][:, :, :, pxc], torch.zeros((), dtype=dtype, device=dev))
    return out


def digit_exponent_t(absmax):
    """digit_exponent() of an fp32 tensor: e with s = 2^(e - 127) > absmax / 127, clamped to [27, 227]."""
    t = absmax.float() / 127.0
    return (((t.view(torch.int32) >> 23) & 0xFF) + 1).clamp(27, 227)


def digits_t(g, e):
    """X = rint(gy 2^24 / s), half to even: the kernel's fp32 product by a power of two (exact) rounded to int."""
    return torch.round(g.double() * pow2(24 + 127 - e)[..., None, None])


def wgrad_t(frames, idx, gp, arg, base=None, chunk=CHUNK):
    """The stem's weight gradient (16, 4, 3, 3) fp32 from rows `idx` of uint8 frames, dL/d(pooled) and the argmax:
    gy folded in fp32, the per-(stack, channel) digit exponent of 4 max|gp|, X = rint(gy 2^24 / s), each stack's
    exact integer sums (every product below 2^39, every sum below 2^53) scaled by s 2^-24, summed over stacks in
    float64, divided by 255, added to `base` in float64 when given, and cast.  The kernel adds the same per-stack terms
    in another float64 order, so it agrees to one fp32 ulp."""
    n, C = gp.shape[:2]
    H, W = frames.shape[-2:]
    total = torch.zeros(C, 36, dtype=torch.float64, device=gp.device)
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        g = fold_t(gp[a:b], arg[a:b], H, W)
        e = digit_exponent_t(4 * gp[a:b].abs().amax(dim=(2, 3)))                # (n, C)
        X = digits_t(g, e).view(b - a, C, H * W)
        S = torch.matmul(X, patches_t(_rows(frames, idx, a, b)).transpose(1, 2))  # (n, C, 36): exact
        total += (S * pow2(e - 127 - 24)[..., None]).sum(0)
    ref = total / 255.0
    if base is not None:
        ref = base.double().reshape(C, 36) + ref
    return ref.float().view(C, 4, 3, 3)


def ulps(a, b):
    """|a - b| in units in the last place of fp32, elementwise (int64), across zero too."""
    def ordered(t):
        i = t.float().contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return (ordered(a) - ordered(b)).abs()
