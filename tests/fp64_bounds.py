"""fp64 references and per-element error bounds of the library's hand-written kernels, shared by the GPU tests that hold
conv_1 (forward and weight gradient), the residual network's stem (forward and weight gradient), the 3xTF32 dense
layers, the dueling tail, V-trace and the fused RMSprop to fp64 at the learners' step shapes (test_gpu_22_step_shapes,
test_gpu_25_apex_step_shapes, test_gpu_35_secondary_steps_fp64, test_gpu_40_impala_resnet,
test_gpu_41_impala_resnet_step_fp64), and the whole-step comparison against an fp64 restatement (check_vs_reference).

Every output element is held to its own bound, computed by the same fp64 reference applied to absolute values
(`mag`), so the bound grows with the length of the sum behind that element; u = 2^-24.  The bound of each kernel is
written in its checker's docstring.  The fp64 references run on the device, a chunk of frame stacks at a time; the
frames are drawn on the device from seeded generators.  Importing this module needs torch, not a GPU;
check_stem, check_stem_wgrad, check_vtrace and check_vs_reference run on tensors of any device."""
import math

import torch

from stem_model import digit_exponent_t, pow2

F = torch.nn.functional

U = 2.0 ** -24
CHUNK = 512                     # frame stacks per fp64 reference chunk (im2col of 512 stacks in fp64: 420 MB)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _frames(n, seed):
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, device="cuda", generator=_gen(seed))


class _Worst:
    """Largest |got - ref| / tol over the chunks of one check, and where it occurs."""

    def __init__(self, what):
        self.what, self.ratio, self.where = what, 0.0, None

    def add(self, got, ref, tol, at=""):
        err = (got.double() - ref).abs()
        r = torch.where(err == 0, torch.zeros_like(err), err / tol).nan_to_num(nan=math.inf)
        k = int(r.argmax())
        v = r.reshape(-1)[k].item()
        if v > self.ratio or self.where is None:
            pos = []
            for s in reversed(r.shape):
                pos.append(k % s)
                k //= s
            pos = tuple(reversed(pos))
            self.ratio = max(v, self.ratio)
            self.where = (at, pos, got.double()[pos].item(), ref[pos].item(), tol[pos].item())

    def check(self):
        print(f"[err/tol] {self.what}: {self.ratio:.3g}")
        assert self.ratio <= 1.0, (f"{self.what}: largest |got - ref| / tol = {self.ratio:.3g} at (chunk, index, got, "
                                   f"ref, tol) = {self.where}")
        return self.ratio


# --------------------------------------------------------------------------- #
# conv_1                                                                        #
# --------------------------------------------------------------------------- #
def check_conv1(what, frames, idx, weights, outs, relu):
    """conv1_fused output `outs[i]` (n, C, 20, 20) of net i against F.conv2d(x / 255, W_i) in fp64, per element
        |got - ref| <= 2^-22 s_c sum_e x_e / 255 + 4u |ref|,      s_c = max|W_c| / 127,
    the first term the four 7-bit digits' truncation |W - s sum_j q_j 2^-7j| <= s 2^-22 times the patch sum, the second
    the fp32 roundings after the exact integer sums (two conversions, one FMA, the scale).  |ref| is the value before
    the ReLU, which can only shrink the difference."""
    n = outs[0].shape[0]
    ones = torch.ones(1, 4, 8, 8, dtype=torch.float64, device="cuda")
    worst = [_Worst(f"{what} net {i}") for i in range(len(weights))]
    wd = [w.double() for w in weights]
    sc = [(w.abs().amax(dim=(1, 2, 3)).float() / 127.0).double().view(1, -1, 1, 1) for w in weights]
    for a in range(0, n, CHUNK):
        b = min(n, a + CHUNK)
        x = (frames[a:b] if idx is None else frames[idx[a:b]]).double() / 255.0
        sx = F.conv2d(x, ones, stride=4)
        for i, o in enumerate(outs):
            ref = F.conv2d(x, wd[i], stride=4)
            tol = 2.0 ** -22 * sc[i] * sx + 4 * U * ref.abs()
            worst[i].add(o[a:b], ref.clamp_min(0) if relu else ref, tol, at=a)
        del x, sx
    return [w.check() for w in worst]


def wgrad_ref(frames, idx, gy, relu_y=None):
    """-> (dW, mag = sum |gy| x, S_e = sum_{k,p} x_e, G_c = max |gy_c|) in fp64, gy masked by relu_y > 0 when given."""
    n, c = gy.shape[:2]
    ref = torch.zeros(c, 256, dtype=torch.float64, device="cuda")
    mag, S = torch.zeros_like(ref), torch.zeros(256, dtype=torch.float64, device="cuda")
    G = torch.zeros(c, dtype=torch.float64, device="cuda")
    for a in range(0, n, CHUNK):
        b = min(n, a + CHUNK)
        x = (frames[a:b] if idx is None else frames[idx[a:b]]).double() / 255.0
        cols = F.unfold(x, 8, stride=4).transpose(1, 2).reshape(-1, 256)          # [(k, p)][e]
        del x
        g = gy[a:b].double()
        if relu_y is not None:
            g = g * (relu_y[a:b] > 0)
        g = g.reshape(b - a, c, 400).transpose(0, 1).reshape(c, -1)               # [c][(k, p)]
        ref += g @ cols
        mag += g.abs() @ cols
        S += cols.sum(0)
        G = torch.maximum(G, g.abs().amax(1))
        del cols, g
    return ref, mag, S, G


def check_wgrad(what, frames, idx, gy, got, base=None, relu_y=None):
    """conv1_wgrad result `got` (C, 4, 8, 8) against base + the fp64 weight gradient, per element
        |got - ref| <= (2 G_c / 127) 2^-25 S_e + 6u mag + 2u |base|,
    G_c = max |gy_c| over all items bounds each CTA's power-of-two digit scale s < 2 G_c / 127, and s 2^-25 is the
    rounding of gy to four base-256 digits; S_e = sum_{k,p} x/255 at patch element e, mag = sum |gy| x/255.  6u: the
    digit recombination (two conversions, one FMA, the scale), the fp32 store of the reduction and the second store
    of a split launch; 2u |base|: the two additions into an existing gradient."""
    ref, mag, S, G = wgrad_ref(frames, idx, gy, relu_y)
    c = ref.shape[0]
    tol = (2.0 * G / 127.0).view(c, 1) * 2.0 ** -25 * S.view(1, 256) + 6 * U * mag
    if base is not None:
        b = base.double().reshape(c, 256)
        ref, tol = ref + b, tol + 2 * U * b.abs()
    w = _Worst(what)
    w.add(got.reshape(c, 256), ref, tol)
    return w.check()


# --------------------------------------------------------------------------- #
# the residual network's stem (csrc/stem.cu)                                    #
# --------------------------------------------------------------------------- #
def _stem_rows(frames, idx, a, b, dev):
    return (frames[a:b] if idx is None else frames[idx[a:b]]).to(dev)


def _stem_unpool(gp, argmax, H, W):
    """The max-pool's backward through `argmax` in fp64 (n, C, H, W): each pooled gradient added at its window's
    chosen position."""
    n, C, PH, PW = gp.shape
    a = argmax.long()
    py = torch.arange(PH, device=gp.device).view(PH, 1)
    px = torch.arange(PW, device=gp.device).view(1, PW)
    pos = ((2 * py - 1 + a // 3) * W + (2 * px - 1 + a % 3)).view(n, C, -1)
    gy = torch.zeros(n, C, H * W, dtype=torch.float64, device=gp.device)
    return gy.scatter_add_(2, pos, gp.double().reshape(n, C, -1)).view(n, C, H, W)


def check_stem(what, frames, idx, weight, pooled, argmax):
    """stem_fused's pooled output and argmax (n, 16, PH, PW) of rows `idx` of uint8 `frames` against the fp64 conv
    ref = F.conv2d(x / 255, W, padding=1), per conv position
        tol = 2^-22 (1 + 2^-8) s_c sum_e x_e / 255 + 6u |ref|,      s_c = max|W_c| / 127,
    sum_e over the zero-padded 3x3 patch.  The first term is the four 7-bit digits' truncation
    |W - s sum_j q_j 2^-7j| <= s 2^-22 times the patch sum; its 2^-8 covers ft's fp32 conversion, which is inexact only
    when |ft| >= 2^24 and then errs by at most 2^-38 |ft| <= 2^-24 sum_e x_e of the digit sums' unit s / (255 * 128),
    below 2^-9 of the first term.  6u |ref|: the fp32 roundings after the exact sums (fu's conversion, inexact only when
    |fu| >= 2^24 >> |ft 2^-14| so within u of |ref|; the FMA; the stored s / 255; the product), plus 1u for the second
    order terms.  The pooled value is the kernel's conv value at its own argmax a, so
        |pooled - ref[a]| <= tol[a],   and   ref[a] + tol[a] >= max_j (ref[j] - tol[j]) over every window's positions j:
    the kernel's maximum is at least each of its window's kernel values.  Every argmax is 3i + j <= 8 and names a
    position inside the frame, never the padding.  -> (pooled value ratio, window ratio)."""
    n = pooled.shape[0]
    dev = pooled.device
    wd = weight.detach().to(dev, torch.float64)
    sc = (weight.detach().abs().amax(dim=(1, 2, 3)).float() / 127.0).to(dev, torch.float64).view(1, -1, 1, 1)
    ones = torch.ones(1, 4, 3, 3, dtype=torch.float64, device=dev)
    held_w, win_w = _Worst(f"{what} pooled value at its argmax"), _Worst(f"{what} window maximum")
    PH, PW = pooled.shape[-2:]
    py = torch.arange(PH, device=dev).view(PH, 1)
    px = torch.arange(PW, device=dev).view(1, PW)
    for a in range(0, n, CHUNK):
        b = min(n, a + CHUNK)
        x = _stem_rows(frames, idx, a, b, dev).double() / 255.0
        ref = F.conv2d(x, wd, padding=1)
        tol = 2.0 ** -22 * (1 + 2.0 ** -8) * sc * F.conv2d(x, ones, padding=1) + 6 * U * ref.abs()
        del x
        H, W = ref.shape[-2:]
        am = argmax[a:b].long()
        assert am.max().item() <= 8, f"{what}: an argmax above 8"
        yy, xx = 2 * py - 1 + am // 3, 2 * px - 1 + am % 3
        assert ((yy >= 0) & (xx >= 0) & (yy < H) & (xx < W)).all(), f"{what}: an argmax names a padded position"
        pos = (yy * W + xx).flatten(2)
        held = ref.flatten(2).gather(2, pos).view_as(am)
        t_held = tol.flatten(2).gather(2, pos).view_as(am)
        del pos, yy, xx, am
        held_w.add(pooled[a:b], held, t_held, at=a)
        lower = F.max_pool2d(ref - tol, 3, 2, 1)                    # max_j (ref[j] - tol[j]), padding skipped
        del ref, tol
        win_w.add(torch.maximum(lower, held), held, t_held, at=a)  # error: how far the window's floor lies above
        del lower, held, t_held
    return held_w.check(), win_w.check()


def check_stem_wgrad(what, frames, idx, gp, argmax, got, base=None):
    """stem_wgrad's result `got` (16, 4, 3, 3) against base + the fp64 weight gradient of the same rows, routed through
    the kernel's `argmax`: ref[c, e] = sum_{n,p} gy[n, c, p] x_e[n, p] / 255 with gy the pool's backward, per element
        tol = 2^-25 sum_n s_{n,c} S_{n,e} + 5u mag + 2u |base|.
    s_{n,c} = 2^(e-127) is the kernel's power-of-two digit scale of stack n, channel c (digit_exponent(4 max|gp|),
    clamped to [27, 227]); rounding gy 2^24 / s to an integer errs by at most 1/2, s 2^-25 in gy, times
    S_{n,e} = sum_p x_e[n, p] / 255, the stack's patch sum of element e over its positions.  mag = the same fp64 weight
    gradient of the fold of |gp|: 3u for the fp32 fold (at most four terms, three roundings), 1u for the fp32 store,
    1u for the fp64 sums over stacks, warps and CTAs (n 2^-53 << u) and the second order terms.  2u |base|: the
    addition into an existing gradient.  The digit sums themselves and their scaling by s 2^-24 are exact."""
    n, C = gp.shape[:2]
    dev = gp.device
    ref = torch.zeros(C, 36, dtype=torch.float64, device=dev)
    mag, D = torch.zeros_like(ref), torch.zeros_like(ref)
    for a in range(0, n, CHUNK):
        b = min(n, a + CHUNK)
        x = _stem_rows(frames, idx, a, b, dev).double() / 255.0
        H, W = x.shape[-2:]
        g, am = gp[a:b], argmax[a:b]
        shape = (C,) + x.shape[1:2] + (3, 3)
        ref += torch.nn.grad.conv2d_weight(x, shape, _stem_unpool(g, am, H, W), padding=1).view(C, 36)
        mag += torch.nn.grad.conv2d_weight(x, shape, _stem_unpool(g.abs(), am, H, W), padding=1).view(C, 36)
        p = F.pad(x, (1, 1, 1, 1))
        S = torch.stack([p[:, :, ky:ky + H, kx:kx + W].sum(dim=(2, 3)) for ky in range(3) for kx in range(3)], 2)
        s = pow2(digit_exponent_t(4 * g.abs().amax(dim=(2, 3))) - 127)                 # (n, C)
        D += 2.0 ** -25 * (s.T @ S.reshape(b - a, 36))
        del x, p
    tol = D + 5 * U * mag
    if base is not None:
        bd = base.double().reshape(C, 36)
        ref, tol = ref + bd, tol + 2 * U * bd.abs()
    w = _Worst(what)
    w.add(got.reshape(C, 36), ref, tol)
    return w.check()


# --------------------------------------------------------------------------- #
# 3xTF32 GEMM                                                                   #
# --------------------------------------------------------------------------- #
def gemm_splits(M, N, K):
    """The K splits b2rl_gemm_tf32x3 uses for C[M][N] = A[M][K] B[N][K]^T (from its workspace size)."""
    from distributed_rl_b200 import _lib
    ldc = (N + 3) // 4 * 4
    n_ws = _lib.load().b2rl_gemm_workspace_floats(M, N, K, ldc)
    return n_ws // (M * ldc) if n_ws else 1


def _rel(c, ref):
    return ((c.double() - ref).abs().max() / ref.abs().max()).item()


def gemm_tol(M, N, K, mag):
    """check_gemm's per-element bound (5 2^-22 + d 2^-23) mag of a [M][K] x [N][K]^T product, `mag` = |a| @ |b|^T in
    fp64."""
    sp = gemm_splits(M, N, K)
    d = 12 * math.ceil(math.ceil(K / 32) / sp) + sp
    return (5 * 2.0 ** -22 + d * 2.0 ** -23) * mag


def check_gemm(what, a, b, got, vs_cublas=4):
    """3xTF32 result `got` = a @ b.T ([M][K] x [N][K]) against fp64, two ways.
    Worst case, per element: |got - ref| <= (5 2^-22 + d 2^-23) mag with mag = |a| @ |b|^T and
    d = 12 ceil(ceil(K/32) / splits) + splits: lo = x - rn_tf32(x) is read by the tensor core truncated to TF32
    (2^-21 relative to x, once per operand) and lo*lo (2^-22) is dropped; each 32-wide K chunk is 3 MMAs x 4 k8 steps
    of fp32 accumulation, then the splits are summed.  That bound would not notice a dropped lo term, so also, as in
    test_gpu_03_gemm: max|err| / max|ref| below `vs_cublas` (4) x cuBLAS fp32's on the same inputs + 5e-7, and below
    plain TF32's / 20."""
    M, K = a.shape
    N = b.shape[0]
    sp = gemm_splits(M, N, K)
    ad, bd = a.double(), b.double()
    ref = ad @ bd.T
    tol = gemm_tol(M, N, K, ad.abs() @ bd.abs().T)
    del ad, bd
    w = _Worst(f"{what} [{M}x{K}]·[{N}x{K}]^T, {sp} split(s)")
    w.add(got, ref, tol)
    del tol
    e3, e32 = _rel(got, ref), _rel(a @ b.T, ref)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        e_tf32 = _rel(a @ b.T, ref)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    print(f"[gemm] {what}: 3xTF32 {e3:.3g}, cuBLAS fp32 {e32:.3g}, TF32 {e_tf32:.3g} (of max|ref|)")
    w.check()
    assert e3 < vs_cublas * e32 + 5e-7, (what, e3, e32, e_tf32)
    if K >= 512 and M > 1:
        assert e3 < e_tf32 / 20, (what, e3, e32, e_tf32)
    return e3, e32, e_tf32


# --------------------------------------------------------------------------- #
# dueling tail                                                                  #
# --------------------------------------------------------------------------- #
def _dueling_nodes(h, wa, wv):
    r = torch.relu(h)
    H = wa.shape[1]
    adv, val = r[:, :H] @ wa.T, r[:, H:] @ wv.T
    return (adv + val) - adv.mean(dim=-1, keepdim=True)


def dueling_forward_tol(h, wa, wv):
    """check_dueling_forward's per-element bound (d + 2) u mag, in fp64 (see there)."""
    A, H = wa.shape
    r = torch.relu(h.double())
    ma = r[:, :H] @ wa.double().abs().T
    mag = ma + r[:, H:] @ wv.double().abs().T + ma.mean(dim=-1, keepdim=True)
    d = H // 32 + 5 + (A - 1) + 2
    return (d + 2) * U * mag


def check_dueling_forward(what, h, wa, wv, q):
    """Dueling forward q against the unfused node sequence in fp64, per element |got - ref| <= (d + 2) u mag, mag the
    node sequence on |wa|, |wv| (relu(h) >= 0 already), d = H/32 + 5 + (A - 1) + 2: one lane's FMA chain, the 5-step
    warp reduction, the sum of the A advantages, the mean's division and the final add and subtract."""
    A, H = wa.shape
    ref = _dueling_nodes(h.double(), wa.double(), wv.double())
    w = _Worst(f"{what} forward, M={h.shape[0]} H={H} A={A}")
    w.add(q, ref, dueling_forward_tol(h, wa, wv))
    return w.check()


def check_dueling_backward(what, h, wa, wv, gq, gh, gwa, gwv):
    """Dueling backward against fp64 autograd of the node sequence, per element |got - ref| <= (d + 2) u mag, mag the
    same backward on absolute values (g_adv -> |gq| + mean |gq|, g_val -> sum |gq|):
    dL/dh: d = A + 5 + 2 (the A-long FMA chain over the advantages, the 5-step warp sum of gq, the mean's division and
    subtraction); dL/dWa, dL/dWv: d = ceil(M/32) + 2 + 8 + 7 (one thread's rows, two shuffles, eight warp partials,
    and the row table's own 7 roundings).  A None gradient is not checked."""
    M, A, H = h.shape[0], wa.shape[0], wa.shape[1]
    hd, wad, wvd = (t.detach().double().requires_grad_() for t in (h, wa, wv))
    _dueling_nodes(hd, wad, wvd).backward(gq.double())
    g = gq.double().abs()
    g_adv = g + g.mean(dim=-1, keepdim=True)
    g_val = g.sum(dim=-1, keepdim=True)
    r = torch.relu(hd.detach())
    on = (hd.detach() > 0).double()
    m_gh = torch.cat([(g_adv @ wad.detach().abs()) * on[:, :H], (g_val @ wvd.detach().abs()) * on[:, H:]], 1)
    m_wa, m_wv = g_adv.T @ r[:, :H], g_val.T @ r[:, H:]
    out = []
    for name, got, ref, mag, d in (("dL/dh", gh, hd.grad, m_gh, A + 5 + 2),
                                   ("dL/dWa", gwa, wad.grad, m_wa, math.ceil(M / 32) + 2 + 8 + 7),
                                   ("dL/dWv", gwv, wvd.grad, m_wv, math.ceil(M / 32) + 2 + 8 + 7)):
        if got is None:
            continue
        w = _Worst(f"{what} {name}, M={M} H={H} A={A}")
        w.add(got, ref, (d + 2) * U * mag)
        out.append(w.check())
    return out


# --------------------------------------------------------------------------- #
# the Ape-X heads: ReLU + NCHW flatten + 3xTF32 GEMM + dueling tail             #
# --------------------------------------------------------------------------- #
def relu_flat(y):
    """flatten_NCHW(relu(y)) of a (B, C, H, W) tensor in any memory format, in fp64: the heads' A operand in the
    weights' feature order c * H * W + p."""
    return torch.relu(y.double()).reshape(y.shape[0], -1)


def check_heads_dueling_forward(what, y, ws, wa, wv, q):
    """q of linear.relu_flat_heads_dueling against dueling(h) in fp64, h = flatten_NCHW(relu(y)) @ cat(ws)^T, per element
        |got - ref| <= tol_duel(h) + tol_h[:, :H] @ |Wa|^T + tol_h[:, H:] @ |Wv|^T + mean_a(tol_h[:, :H] @ |Wa|^T),
    tol_duel the dueling-forward bound of check_dueling_forward evaluated on the fp64 h, tol_h = gemm_tol(M, 2H, K,
    flatten_NCHW(relu(y)) @ |cat(ws)|^T) the 3xTF32 GEMM's bound on each element of the h the kernel sums from the
    split partials.  ReLU is 1-Lipschitz, so an error e in h moves adv by at most e[:, :H] @ |Wa|^T, val by
    e[:, H:] @ |Wv|^T and the advantages' mean by the mean of the first: to first order the three propagated terms."""
    a = relu_flat(y)
    w = torch.cat([t.double() for t in ws], 0)
    M, K = a.shape
    N, (A, H) = w.shape[0], wa.shape
    h = a @ w.T
    tol_h = gemm_tol(M, N, K, a @ w.abs().T)
    del a, w
    e_adv = tol_h[:, :H] @ wa.double().abs().T
    tol = (dueling_forward_tol(h, wa, wv) + e_adv + tol_h[:, H:] @ wv.double().abs().T
           + e_adv.mean(dim=-1, keepdim=True))
    worst = _Worst(f"{what} q, M={M} K={K} N={N} H={H} A={A}")
    worst.add(q, _dueling_nodes(h, wa.double(), wv.double()), tol)
    return worst.check()


def check_relu_flat_dgrad(what, y, ws, gh, gy):
    """dL/dy of h = flatten_NCHW(relu(y)) @ cat(ws)^T (y (M, C, H, W), pre-ReLU) against fp64: unflatten_NCHW(gh @ cat(ws))
    where y > 0 and exactly 0 elsewhere, per element gemm_tol(M, K, N, |gh| @ |cat(ws)|) masked alike.  The dL/dx GEMM
    contracts over N = 2H and b2rl_unflatten_relu_mask sums its split partials in split order, as the GEMM's own
    reduction does, so check_gemm's bound holds as it stands."""
    M = y.shape[0]
    w = torch.cat([t.double() for t in ws], 0)
    N, K = w.shape
    g = gh.double()
    mask = (y.double() > 0).reshape(M, -1)
    ref = (g @ w) * mask
    tol = gemm_tol(M, K, N, g.abs() @ w.abs()) * mask
    worst = _Worst(f"{what} dL/dy [{M}x{N}]·[{N}x{K}], {gemm_splits(M, K, N)} split(s)")
    worst.add(gy.reshape(M, -1), ref, tol)
    return worst.check()


# --------------------------------------------------------------------------- #
# the fused centered RMSprop                                                    #
# --------------------------------------------------------------------------- #
def check_rmsprop_centered(what, pre, post, lr, alpha, eps):
    """One centered RMSprop update of the fused optimizer (csrc/optim.cu rmsprop_elem) against fp64, per element, from
    the tensors the launch read (`pre`: p, g, sq, ga) and wrote (`post`: p, sq, ga, g).  The hyper-parameters are the
    fp32 values the kernel receives (a = alpha, b = 1 - alpha formed in double, lr, eps); the reference is
        S = a sq + b g^2,   G = ga + b (g - ga),   D = S - G^2,   P = p - s,   s = lr g / (sqrt(D) + eps).
    The kernel rounds each operation once (u = 2^-24; -fmad=false, its FMAs are explicit):
      sq' = fma(fl(b g), g, fl(sq a)): two non-negative products rounded once each, then their sum:
            |sq' - S| <= ((1 + u)^2 - 1) S <= 3u S =: t_s;
      ga' = fma(b, fl(g - ga), ga):  |ga' - G| <= u b |g - ga| (1 + u) + u |G| <= u (2 b |g - ga| + |G|) =: t_g;
      D'  = fma(-ga', ga', sq'):     |D' - D| <= t_s + 2 |G| t_g + t_g^2 + u |D'|: relative r_D = (t_s + 2 |G| t_g +
            t_g^2) / D + 2u, the cancellation term, of order u (S + G^2) / D;
      avg = sqrt(D'): r_D / 2 + u;  avg + eps: r_D / 2 + 2u (eps exact, both terms non-negative);  g / ., lr * .:
            r_D / 2 + 4u on the step s;
      p'  = fl(p - s'):              |p' - P| <= |s| (r_D / 2 + 5u) + u |P|,
    one u of slack on the step for the second-order terms (r_D stays near 1e-6 here).  Where the averages and g are all
    zero, D = 0 and s = 0: p' must equal p.  The gradient must read zero after the launch."""
    import numpy as np
    a, b = float(np.float32(alpha)), float(np.float32(1.0 - alpha))
    lr, eps = float(np.float32(lr)), float(np.float32(eps))
    p, g, sq, ga = (pre[k].double() for k in ("p", "g", "sq", "ga"))
    S = a * sq + b * g * g
    G = ga + b * (g - ga)
    D = S - G * G
    s = lr * g / (D.clamp_min(0).sqrt() + eps)
    P = p - s
    t_s = 3 * U * S
    t_g = U * (2 * b * (g - ga).abs() + G.abs())
    r_D = torch.where(D > 0, (t_s + 2 * G.abs() * t_g + t_g * t_g) / D.where(D > 0, torch.ones_like(D)), 0.0) + 2 * U
    out = []
    for name, got, ref, tol in (("square_avg", post["sq"], S, t_s), ("grad_avg", post["ga"], G, t_g),
                                ("param", post["p"], P, s.abs() * (r_D / 2 + 5 * U) + U * P.abs())):
        w = _Worst(f"{what} {name}")
        w.add(got, ref, tol)
        out.append(w.check())
    assert not post["g"].any(), f"{what}: the gradient is not zero after the update"
    return out


# --------------------------------------------------------------------------- #
# V-trace                                                                       #
# --------------------------------------------------------------------------- #
def _f32(x):
    import numpy as np
    return float(np.float32(x))


def vtrace_inputs(T, B, seed):
    """fp32 (pi, mu, value, boot, reward) numpy arrays for V-trace at its edges: pi from 1e-30 to 1 (half of it in
    [0.05, 1], a tenth equal to mu, pi[0, 0] = 1), mu in [1e-3, 0.9], so that pi / mu lies far above and below any
    clip; 30 % of the bootstraps zero."""
    import numpy as np
    rng = np.random.default_rng(seed)
    f32 = np.float32
    pi = (10.0 ** rng.uniform(-30, 0, size=(T, B))).astype(f32)
    mid = rng.random((T, B)) < 0.5
    pi[mid] = rng.uniform(0.05, 1.0, size=int(mid.sum())).astype(f32)
    mu = (10.0 ** rng.uniform(-3, np.log10(0.9), size=(T, B))).astype(f32)
    same = rng.random((T, B)) < 0.1
    pi[same] = mu[same]
    pi[0, 0] = 1.0
    v = rng.standard_normal((T, B)).astype(f32)
    boot = (rng.standard_normal(B) * (rng.random(B) > 0.3)).astype(f32)
    r = rng.standard_normal((T, B)).astype(f32)
    return pi, mu, v, boot, r


def vtrace_ref(pi, mu, value, boot, reward, gamma, lam, cbar, pbar):
    """-> (vt, adv, tol_vt, tol_adv) in fp64: V-trace as csrc/targets.cu k_vtrace and oracle.vtrace compute it (the
    last step not rho-clipped, c_bar both the delta weight and the trace), and check_vtrace's per-element bounds."""
    g, lam, cbar, pbar = (_f32(x) for x in (gamma, lam, cbar, pbar))
    pi, mu, v, r, bs = (t.double() for t in (pi, mu, value, reward, boot))
    T = v.shape[0]
    lp, lm = pi.log(), mu.log()
    ratio = (lp - lm).exp()
    rho = 9 * U * (lp.abs() + lm.abs()) + 7 * U
    cr, pt = ratio.clamp(max=cbar), ratio.clamp(max=pbar)
    e_c, e_p = rho * cr, rho * pt
    vt, adv, t_vt, t_adv = (torch.empty_like(v) for _ in range(4))
    zero = torch.zeros_like(bs)
    vmt_n, e_vmt_n, vt_n, e_vt_n, v_n = zero, zero, bs, zero, zero
    for i in reversed(range(T)):
        nxt = bs if i == T - 1 else v_n
        td = r[i] + g * nxt - v[i]
        e_td = 3 * U * (r[i].abs() + g * nxt.abs() + v[i].abs())
        if i == T - 1:
            vmt, e_vmt = td, e_td
        else:
            t1, t2 = td * cr[i], g * lam * cr[i] * vmt_n
            vmt = t1 + t2
            e_vmt = (td.abs() * e_c[i] + cr[i] * e_td + U * t1.abs()
                     + g * lam * (cr[i] * e_vmt_n + vmt_n.abs() * (e_c[i] + 3 * U * cr[i]))
                     + U * (t1.abs() + t2.abs()))
        vt[i] = v[i] + vmt
        e_vt = e_vmt + U * (v[i].abs() + vmt.abs())
        at = r[i] + g * vt_n
        d = at - v[i]
        e_d = g * e_vt_n + U * (g * vt_n.abs() + at.abs() + d.abs())
        adv[i] = d * pt[i]
        t_vt[i], t_adv[i] = e_vt, pt[i] * e_d + d.abs() * e_p[i] + U * adv[i].abs()
        vmt_n, e_vmt_n, vt_n, e_vt_n, v_n = vmt, e_vmt, vt[i], e_vt, v[i]
    return vt, adv, t_vt, t_adv


def check_vtrace(what, pi, mu, value, boot, reward, gamma, lam, cbar, pbar, vt, adv):
    """V-trace targets `vt` and advantages `adv` (T, B) of fp32 inputs against fp64, per element.  The parameters are
    the fp32 values the kernel receives; every operation of the kernel is rounded once (u = 2^-24).
    The ratio expf(logf(pi) - logf(mu)): logf within 4 ulp (2^-23 |ln x| each), the subtraction within u, so the
    exponent errs by 8u (|ln pi| + |ln mu|) + u |ln pi - ln mu|; expf within 3 ulp.  Relative to pi / mu:
        rho = 9u (|ln pi| + |ln mu|) + 7u
    (4 and 3 ulp cover numpy's float32 log and exp as well as CUDA's logf and expf, 1 and 2 ulp).  The clips
    min(c, ratio) and min(p, ratio) are 1-Lipschitz: e_c = rho min(ratio, c), e_p = rho min(ratio, p).
    td = r + g v' - v errs by 3u (|r| + g |v'| + |v|) =: e_td (v' the next value, the bootstrap at T - 1).  The
    recursion vmt = td cr + (g (lam cr)) vmt' carries its error by the same recursion on absolute values with factor
    g lam cr:
        e_vmt = |td| e_c + cr e_td + u |td cr| + g lam (cr e_vmt' + |vmt'| (e_c + 3u cr)) + u (|td cr| + |g lam cr vmt'|),
    e_vmt = e_td at T - 1 (no ratio there).  vt = v + vmt: e_vt = e_vmt + u (|v| + |vmt|).  adv = ((r + g vt') - v) pt
    with vt' the next target (the bootstrap, exact, at T - 1), at = r + g vt' and d = at - v: three roundings,
    e_d = g e_vt' + u (g |vt'| + |at| + |d|), and e_adv = pt e_d + |d| e_p + u |adv|.  First order in u; the bounds keep 1u of slack per ratio for the rest."""
    ref_vt, ref_adv, t_vt, t_adv = vtrace_ref(pi, mu, value, boot, reward, gamma, lam, cbar, pbar)
    T, B = ref_vt.shape
    out = []
    for name, got, ref, tol in (("vtarget", vt, ref_vt, t_vt), ("advantage", adv, ref_adv, t_adv)):
        w = _Worst(f"{what} {name}, T={T} B={B}")
        w.add(got, ref, tol)
        out.append(w.check())
    return out


# --------------------------------------------------------------------------- #
# a whole step against the fp64, fp32 and TF32 restatements                    #
# --------------------------------------------------------------------------- #
def rel_err(x, ref64):
    """max |x - ref64| / max |ref64| (the absolute error where ref64 is all zero)."""
    err = (x.double() - ref64).abs().max().item()
    den = ref64.abs().max().item()
    return err / den if den > 0 else err


def check_vs_reference(what, got, ref64, ref32, reftf32, k=16, floor=1e-6, sharp=True):
    """A learner step's tensor `got` against the same tensor of an fp64 restatement of the step (`ref64`), with
    e(x) = max |x - ref64| / max |ref64|:
        e(got) <= k e(ref32) + floor      no less accurate than the reference's own fp32 arithmetic, within k;
        e(got) <= e(reftf32) / 20         the comparison is sharp enough to see a TF32-class fault.
    `ref32`, `reftf32`: the restatement in fp32 and with TF32 convolutions and matmuls.  sharp=False drops the second
    test, for a quantity TF32's roundings average out in (the caller says why).  -> (e(got), e(ref32), e(reftf32))."""
    ref64 = ref64.double()
    e, e32, etf = rel_err(got, ref64), rel_err(ref32, ref64), rel_err(reftf32, ref64)
    ratio = e / e32 if e32 > 0 else (0.0 if e == 0 else math.inf)
    print(f"[err/ref] {what}: {e:.3g} of max|ref64|, fp32 {e32:.3g} ({ratio:.3g}x), TF32 {etf:.3g}")
    assert e <= k * e32 + floor, f"{what}: {e:.3g} of max|ref64| exceeds {k} x fp32's {e32:.3g} + {floor:g}"
    assert e <= etf / 20 or not sharp, f"{what}: {e:.3g} of max|ref64| is not below TF32's {etf:.3g} / 20"
    return e, e32, etf
