"""conv_1 (forward and weight gradient), the 3xTF32 dense layers and the dueling tail against fp64 at the shapes the
R2D2 (B = 64, T = 80, MEM = 20) and IMPALA (B = 1024, T = 20) learner steps run them, first on synthetic inputs, then on
the inputs of one real eager step of each learner.

Every output element is held to its own bound, computed by the same fp64 reference applied to absolute values
(`mag`), so the bound grows with the length of the sum behind that element; u = 2^-24.  The bound of each kernel is
written in its checker's docstring.  The fp64 references run on the device, a chunk of frame stacks at a time; the
frames are drawn on the device from seeded generators."""
import math

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = torch.nn.functional

U = 2.0 ** -24
CHUNK = 512                     # frame stacks per fp64 reference chunk (im2col of 512 stacks in fp64: 420 MB)
GY_LIMIT = -0x7E808080 * 2.0 ** -24     # = -126.50196075439453, exact in fp32: digits (-126, -128, -128, -128)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    free, _ = torch.cuda.mem_get_info()
    if free < 20 << 30:
        pytest.skip(f"needs about 16 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def R(dev):
    from distributed_rl_b200 import replay
    return replay


@pytest.fixture(scope="module")
def L(dev):
    from distributed_rl_b200 import linear
    return linear


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


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
# fp64 references and per-element bounds                                       #
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


def gemm_splits(M, N, K):
    """The K splits b2rl_gemm_tf32x3 uses for C[M][N] = A[M][K] B[N][K]^T (from its workspace size)."""
    from distributed_rl_b200 import _lib
    ldc = (N + 3) // 4 * 4
    n_ws = _lib.load().b2rl_gemm_workspace_floats(M, N, K, ldc)
    return n_ws // (M * ldc) if n_ws else 1


def _rel(c, ref):
    return ((c.double() - ref).abs().max() / ref.abs().max()).item()


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
    d = 12 * math.ceil(math.ceil(K / 32) / sp) + sp
    ad, bd = a.double(), b.double()
    ref = ad @ bd.T
    tol = (5 * 2.0 ** -22 + d * 2.0 ** -23) * (ad.abs() @ bd.abs().T)
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


def _dueling_nodes(h, wa, wv):
    r = torch.relu(h)
    H = wa.shape[1]
    adv, val = r[:, :H] @ wa.T, r[:, H:] @ wv.T
    return (adv + val) - adv.mean(dim=-1, keepdim=True)


def check_dueling_forward(what, h, wa, wv, q):
    """Dueling forward q against the unfused node sequence in fp64, per element |got - ref| <= (d + 2) u mag, mag the
    node sequence on |wa|, |wv| (relu(h) >= 0 already), d = H/32 + 5 + (A - 1) + 2: one lane's FMA chain, the 5-step
    warp reduction, the sum of the A advantages, the mean's division and the final add and subtract."""
    A, H = wa.shape
    hd, wad, wvd = h.double(), wa.double(), wv.double()
    ref = _dueling_nodes(hd, wad, wvd)
    r = torch.relu(hd)
    ma = r[:, :H] @ wad.abs().T
    mag = ma + r[:, H:] @ wvd.abs().T + ma.mean(dim=-1, keepdim=True)
    d = H // 32 + 5 + (A - 1) + 2
    w = _Worst(f"{what} forward, M={h.shape[0]} H={H} A={A}")
    w.add(q, ref, (d + 2) * U * mag)
    return w.check()


def check_dueling_backward(what, h, wa, wv, gq, gh, gwa, gwv):
    """Dueling backward against fp64 autograd of the node sequence, per element |got - ref| <= (d + 2) u mag, mag the
    same backward on absolute values (g_adv -> |gq| + mean |gq|, g_val -> sum |gq|):
    dL/dh: d = A + 5 + 2 (the A-long FMA chain over the advantages, the 5-step warp sum of gq, the mean's division and
    subtraction); dL/dWa, dL/dWv: d = ceil(M/32) + 2 + 8 + 7 (one thread's rows, two shuffles, eight warp partials,
    and the row table's own 7 roundings)."""
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
        w = _Worst(f"{what} {name}, M={M} H={H} A={A}")
        w.add(got, ref, (d + 2) * U * mag)
        out.append(w.check())
    return out


# --------------------------------------------------------------------------- #
# A. the kernels at the step shapes, synthetic inputs                          #
# --------------------------------------------------------------------------- #
def _conv1_weights(n_nets, c_out, seed):
    ws = [torch.empty(c_out, 4, 8, 8, device="cuda").uniform_(-0.0625, 0.0625, generator=_gen(seed + i))
          for i in range(n_nets)]
    ws[0][3] = 0.0                                   # an all-zero output channel
    ws[0][5, 0, 0, 0] = 0.9                          # one dominant weight: the small digits of the others matter
    return ws


def _pack(R, ws, c_out):
    pack = R.Conv1Pack(len(ws), "cuda:0", c_out=c_out)
    for i, w in enumerate(ws):
        pack.pack(i, w)
    return pack


def test_conv1_forward_r2d2_time_major_rows(R):
    """R2D2: a table of 64 sequences x 80 frame stacks, time-major rows slot * 80 + t with repeated slots (the payload
    pool's reuse); online + target nets of 32 channels in one launch over the 1 280 burn-in rows (ReLU) and the 3 840
    window rows (no ReLU)."""
    from distributed_rl_b200.learner_common import time_major_rows
    B, T, MEM = 64, 80, 20
    frames = _frames(B * T, 1)
    frames[0, :, :8, :8] = 255                       # saturated corner, read by slot 0's t = 0 burn-in row
    slots = torch.randint(0, B, (B,), device="cuda", generator=_gen(2))
    slots[:3] = torch.tensor([0, 7, 7])              # slot 0 drawn, slot 7 twice
    rows = time_major_rows(slots, torch.arange(T, device="cuda").view(T, 1))
    assert rows.numel() == B * T and int(rows[0]) == 0
    ws = _conv1_weights(2, 32, 10)
    pack = _pack(R, ws, 32)
    for sel, relu in ((rows[:MEM * B], True), (rows[MEM * B:], False)):
        outs = R.conv1_fused(frames, sel, pack, relu=relu)
        assert outs[0].shape == (sel.numel(), 32, 20, 20)
        check_conv1(f"conv1_fused R2D2 n={sel.numel()} relu={relu}", frames, sel, ws, outs, relu)
        assert (outs[0][:, 3] == 0).all()


@pytest.mark.parametrize("shuffled", [False, True])
def test_conv1_forward_impala_all_rollout_frames(R, shuffled):
    """IMPALA: one 16-channel net over all (T + 1) x B = 21 504 frame stacks, in order (idx None) or shuffled."""
    n = 21 * 1024
    frames = _frames(n, 3)
    frames[0, :, :8, :8] = 255
    idx = torch.randperm(n, device="cuda", generator=_gen(4)) if shuffled else None
    ws = _conv1_weights(1, 16, 20)
    outs = R.conv1_fused(frames, idx, _pack(R, ws, 16), relu=False)
    check_conv1(f"conv1_fused IMPALA n={n} shuffled={shuffled}", frames, idx, ws, outs, False)
    assert (outs[0][:, 3] == 0).all()


def _wgrad_gy(n, c_out, seed):
    """dL/dy spread over six decades across items, half of its entries zero, one all-zero channel, one dominant entry."""
    g = _gen(seed)
    gy = torch.randn(n, c_out, 20, 20, device="cuda", generator=g)
    gy *= torch.logspace(-6, 0, n, device="cuda")[torch.randperm(n, device="cuda", generator=g)].view(n, 1, 1, 1)
    gy *= torch.rand(n, c_out, 20, 20, device="cuda", generator=g) > 0.5
    gy[:, 3] = 0.0
    gy[0, 5, 0, 0] = 50.0
    return gy.contiguous(memory_format=torch.channels_last)


def test_conv1_wgrad_r2d2_window_rows(R):
    """R2D2: the weight gradient of the 3 840 window rows (time-major, through idx), 32 channels."""
    from distributed_rl_b200.learner_common import time_major_rows
    B, T, MEM = 64, 80, 20
    frames = _frames(B * T, 5)
    frames[1] = 255
    slots = torch.randint(0, B, (B,), device="cuda", generator=_gen(6))
    rows = time_major_rows(slots, torch.arange(T, device="cuda").view(T, 1))[MEM * B:].contiguous()
    gy = _wgrad_gy(rows.numel(), 32, 7)
    gw = R.conv1_wgrad(frames, rows, gy)
    check_wgrad(f"conv1_wgrad R2D2 n={rows.numel()}", frames, rows, gy, gw)
    assert (gw[3] == 0).all()


def test_conv1_wgrad_impala_rows_in_order(R):
    """IMPALA: the weight gradient of the T x B = 20 480 sequence rows read in order (idx None), 16 channels."""
    n = 20 * 1024
    frames = _frames(n, 8)
    frames[0] = 255
    gy = _wgrad_gy(n, 16, 9)
    gw = R.conv1_wgrad(frames, None, gy)
    check_wgrad(f"conv1_wgrad IMPALA n={n}", frames, None, gy, gw)
    assert (gw[3] == 0).all()


@pytest.mark.parametrize("with_idx,accumulate", [(False, False), (True, False), (False, True), (True, True)])
def test_conv1_wgrad_split_over_two_launches(R, sms, with_idx, accumulate):
    """n = SMs * 160 + 257 items: more than one launch's worth at MAX_ITEMS_PER_CTA = 160, so the second launch reads gy,
    y and the frames (idx None) at the item offset and adds to the first launch's result; with `accumulate` both add
    to a non-zero gradient."""
    n = sms * 160 + 257
    rows = 4096 if with_idx else n
    frames = _frames(rows, 11)
    idx = torch.randint(0, rows, (n,), device="cuda", generator=_gen(12)) if with_idx else None
    gy = _wgrad_gy(n, 32, 13)
    y = torch.relu(torch.randn(n, 32, 20, 20, device="cuda", generator=_gen(14))).contiguous(
        memory_format=torch.channels_last)
    base = torch.randn(32, 4, 8, 8, device="cuda", generator=_gen(15)) if accumulate else None
    out = base.clone() if accumulate else torch.full((32, 4, 8, 8), float("nan"), device="cuda")
    R.conv1_wgrad(frames, idx, gy, out=out, accumulate=accumulate, relu_y=y)
    check_wgrad(f"conv1_wgrad split n={n} idx={with_idx} accumulate={accumulate}", frames, idx, gy, out, base=base,
                relu_y=y)


@pytest.mark.parametrize("items", ["160", "160+1", "200"])
def test_conv1_wgrad_accumulators_at_their_limit(R, sms, items):
    """Every pixel 255 and gy = -0x7E808080 * 2^-24 in every channel: with its digit scale of 1 each gy splits into the
    digits (-126, -128, -128, -128), so every int32 column sum of a CTA holding 160 items is -128 * 255 * 400 * 160,
    3 % inside int32.  dW = n * 400 * gy exactly (x / 255 = 1); an overflow flips a sign.  n = SMs * 160 fills every
    CTA to the limit, SMs * 160 + 1 adds a one-item second launch, SMs * 200 would put 200 items in a CTA if it ran
    as one launch."""
    n = {"160": sms * 160, "160+1": sms * 160 + 1, "200": sms * 200}[items]
    frames = torch.full((n, 4, 84, 84), 255, dtype=torch.uint8, device="cuda")
    gy = torch.full((n, 20, 20, 32), GY_LIMIT, device="cuda").permute(0, 3, 1, 2)      # channels_last
    assert gy.is_contiguous(memory_format=torch.channels_last) and gy[0, 0, 0, 0].item() == GY_LIMIT
    gw = R.conv1_wgrad(frames, None, gy)
    want = n * 400 * GY_LIMIT
    rel = ((gw.double() - want).abs() / abs(want)).max().item()
    print(f"[err/tol] conv1_wgrad at the int32 limit n={n}: {rel / 1e-6:.3g}")
    assert rel <= 1e-6, (n, gw.min().item(), gw.max().item(), want)


def _heads_case(case):
    g = _gen({"r2d2": 21, "impala": 22, "impala_boot": 23}[case])
    if case == "r2d2":       # the LSTM output: signed, in (-1, 1); advantage | value first layers, 512 each
        M, K, Ns = 3840, 512, (512, 512)
        x = torch.tanh(torch.randn(M, K, device="cuda", generator=g))
    else:                    # the ReLU'd conv stack: non-negative, about half zeros; one 256-wide layer
        M, K, Ns = (20480 if case == "impala" else 1024), 2592, (256,)
        x = torch.relu(torch.randn(M, K, device="cuda", generator=g))
    x[0, 0] = 1e4                                    # wide dynamic range within a row
    ws = [torch.empty(n, K, device="cuda").uniform_(-K ** -0.5, K ** -0.5, generator=g) for n in Ns]
    gy = torch.randn(M, sum(Ns), device="cuda", generator=g) * (torch.rand(M, sum(Ns), device="cuda", generator=g) > 0.5)
    gy *= 1e-3 if case == "r2d2" else 1.0 / (20 * 1024)
    return x, ws, gy


@pytest.mark.parametrize("case", ["r2d2", "impala", "impala_boot"])
def test_heads_3xtf32_forward_and_backward(L, case):
    """linear3x forward, dL/dx and dL/dW: R2D2's [3840, 512] x [512 | 512] (stacked pair), IMPALA's [20480, 2592] x
    [256] (weight gradient K = 20 480) and its [1024, 2592] bootstrap pass.
    R2D2's dL/dx is held to 8x cuBLAS fp32 instead of 4x.  Measured on an H100 SXM (132 SMs, 700 W): 3xTF32 3.7e-6 of
    max|ref| there, about what it errs on Ape-X's dL/dx with the same 16-chunk splits (4.4e-6, 2.7x cuBLAS), but
    cuBLAS fp32 picks a more accurate kernel for this shape (5.2e-7, 1.6e-6 at Ape-X's): 7.1x.  8-chunk splits bring
    it to 3.2x and slow the Ape-X step by 7 %."""
    x, ws, gy = _heads_case(case)
    xg = x.clone().requires_grad_()
    wg = [w.clone().requires_grad_() for w in ws]
    y = L.linear3x(xg, wg if len(wg) > 1 else wg[0])
    w = torch.cat(ws, 0)
    check_gemm(f"{case} forward", x, w, y.detach())
    del y
    if case == "impala_boot":
        return
    L.linear3x(xg, wg if len(wg) > 1 else wg[0]).backward(gy)
    check_gemm(f"{case} dL/dx", gy, w.T.contiguous(), xg.grad, vs_cublas=8 if case == "r2d2" else 4)
    check_gemm(f"{case} dL/dW", gy.T.contiguous(), x.T.contiguous(), torch.cat([t.grad for t in wg], 0))


def test_dueling_tail_r2d2_forward_and_backward(L):
    """linear.dueling_tail forward, dL/dh, dL/dWa and dL/dWv at R2D2's M = 3 840, H = 512, A = 6: the weight gradient
    kernel sums 120 rows per thread."""
    M, H, A = 3840, 512, 6
    g = _gen(32)
    h = (torch.randn(M, 2 * H, device="cuda", generator=g) * 0.3).requires_grad_()
    wa = (torch.randn(A, H, device="cuda", generator=g) * 0.05).requires_grad_()
    wv = (torch.randn(1, H, device="cuda", generator=g) * 0.05).requires_grad_()
    gq = torch.randn(M, A, device="cuda", generator=g) * 1e-2
    q = L.dueling_tail(h, wa, wv)
    q.backward(gq)
    check_dueling_forward("dueling_tail R2D2", h.detach(), wa.detach(), wv.detach(), q.detach())
    check_dueling_backward("dueling_tail R2D2", h, wa, wv, gq, h.grad, wa.grad, wv.grad)


def test_dueling_tail_r2d2_partials(L):
    """R2D2's tail (M = 3 840, H = 512, A = 6) fed three K-split partials of h, the way the fused heads + tail op hands
    them over: the kernel sums them in split order (h_out equals that fp32 sum bit for bit) before the tail."""
    from distributed_rl_b200 import _lib
    M, H, A, S = 3840, 512, 6, 3
    g = _gen(31)
    stride = M * 2 * H + 64                          # partials need not be packed back to back
    part = torch.randn(S * stride, device="cuda", generator=g) * 0.3
    views = [part[z * stride: z * stride + M * 2 * H].view(M, 2 * H) for z in range(S)]
    wa = torch.randn(A, H, device="cuda", generator=g) * 0.05
    wv = torch.randn(1, H, device="cuda", generator=g) * 0.05
    q = torch.empty(M, A, device="cuda")
    h = torch.empty(M, 2 * H, device="cuda")
    _lib.check(_lib.load().b2rl_dueling_forward(part.data_ptr(), S, stride, M, H, wa.data_ptr(), A, wv.data_ptr(),
                                                q.data_ptr(), h.data_ptr(), torch.cuda.current_stream().cuda_stream))
    assert torch.equal(h, (views[0] + views[1]) + views[2])
    check_dueling_forward("dueling_tail R2D2 from 3 partials", h, wa, wv, q)


# --------------------------------------------------------------------------- #
# B. the same kernels on one real eager step of each learner                   #
# --------------------------------------------------------------------------- #
class _Spies:
    """Record the inputs and outputs of conv1_fused, conv1_wgrad, linear3x and dueling_tail (forward) during a step;
    Conv1Pack.pack records the weights each pack holds.  `out` of conv1_wgrad is copied before the call: in the
    deferred-gradient mode the kernel accumulates into .grad."""

    def __init__(self, monkeypatch, R, L):
        self.calls = {"conv1_fused": [], "conv1_wgrad": [], "linear3x": [], "dueling_tail": []}
        self.packed = {}
        orig_pack, orig_fused, orig_wgrad = R.Conv1Pack.pack, R.conv1_fused, R.conv1_wgrad
        orig_lin, orig_duel = L.linear3x, L.dueling_tail

        def pack(p, net, weight):
            self.packed[(id(p), net)] = weight.detach().float().clone()
            return orig_pack(p, net, weight)

        def conv1_fused(frames, idx, p, relu=False, out=None):
            res = orig_fused(frames, idx, p, relu=relu, out=out)
            self.calls["conv1_fused"].append(dict(
                frames=frames, idx=None if idx is None else idx.clone(), relu=relu,
                weights=[self.packed[(id(p), i)] for i in range(p.n_nets)], outs=[o.clone() for o in res]))
            return res

        def conv1_wgrad(frames, idx, gy, out=None, accumulate=False, relu_y=None):
            base = out.clone() if (out is not None and accumulate) else None
            res = orig_wgrad(frames, idx, gy, out=out, accumulate=accumulate, relu_y=relu_y)
            self.calls["conv1_wgrad"].append(dict(
                frames=frames, idx=None if idx is None else idx.clone(), gy=gy.detach().clone(), base=base,
                relu_y=None if relu_y is None else relu_y.detach().clone(), got=res.detach().clone()))
            return res

        def linear3x(x, w, cache=None):
            y = orig_lin(x, w, cache)
            ws = [w] if torch.is_tensor(w) else list(w)
            self.calls["linear3x"].append(dict(x=x.detach().clone(), w=torch.cat([t.detach() for t in ws], 0),
                                               y=y.detach().clone()))
            return y

        def dueling_tail(h, wa, wv):
            q = orig_duel(h, wa, wv)
            self.calls["dueling_tail"].append(dict(h=h.detach().clone(), wa=wa.detach().clone(),
                                                   wv=wv.detach().clone(), q=q.detach().clone()))
            return q

        monkeypatch.setattr(R.Conv1Pack, "pack", pack)
        monkeypatch.setattr(R, "conv1_fused", conv1_fused)
        monkeypatch.setattr(R, "conv1_wgrad", conv1_wgrad)
        monkeypatch.setattr(L, "linear3x", linear3x)
        monkeypatch.setattr(L, "dueling_tail", dueling_tail)

    def check(self, what, R):
        for c in self.calls["conv1_fused"]:
            check_conv1(f"{what} conv1_fused n={c['outs'][0].shape[0]} relu={c['relu']}", c["frames"], c["idx"],
                        c["weights"], c["outs"], c["relu"])
        for c in self.calls["conv1_wgrad"]:
            check_wgrad(f"{what} conv1_wgrad n={c['gy'].shape[0]}", c["frames"], c["idx"], c["gy"], c["got"],
                        base=c["base"], relu_y=c["relu_y"])
        for c in self.calls["linear3x"]:
            check_gemm(f"{what} linear3x", c["x"], c["w"], c["y"])
        for c in self.calls["dueling_tail"]:
            check_dueling_forward(f"{what} dueling_tail", c["h"], c["wa"], c["wv"], c["q"])


def test_one_r2d2_step_at_the_bench_shapes(R, L, monkeypatch):
    """bench.py's R2D2 line (B = 64, T = 80, MEM = 20) on a 256-sequence replay filled the way bench.py fills it: every
    conv_1, conv_1 weight gradient, heads GEMM and dueling tail of one eager fused step against fp64."""
    from distributed_rl_b200 import r2d2
    B, T, N = 64, 80, 256
    cfg = r2d2.R2D2Config(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, FIXED_TRAJECTORY=T, MEM=20,
                          LEARNER_DEVICE="cuda:0")
    torch.manual_seed(0)
    lrn = r2d2.Learner(cfg, start_replay=False)
    st = lrn.memory.store
    g = _gen(0xB207)
    st.fill_hash(N, seed=0xB203)
    st.field_view("action").copy_(torch.randint(0, 6, (N, T), device="cuda", generator=g, dtype=torch.int32))
    st.field_view("reward").copy_(torch.randn(N, T, device="cuda", generator=g))
    st.field_view("h0").copy_(torch.randn(N, 512, device="cuda", generator=g) * 0.1)
    st.field_view("h1").copy_(torch.randn(N, 512, device="cuda", generator=g) * 0.1)
    st.field_view("notdone").copy_((torch.rand(N, device="cuda", generator=g) > 0.02).float())
    st.build((torch.randn(N, device="cuda", generator=g).abs().clamp(max=1) + 1e-7) ** cfg.ALPHA)
    st.seed(1234, 0)
    spies = _Spies(monkeypatch, R, L)
    lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    n = {k: len(v) for k, v in spies.calls.items()}
    assert n["conv1_fused"] == 2 and n["conv1_wgrad"] == 1 and n["linear3x"] >= 2 and n["dueling_tail"] >= 2, n
    spies.check("R2D2 step", R)
    st.close()


def test_one_impala_step_at_the_bench_shapes(R, L, monkeypatch):
    """bench.py's IMPALA line (B = 1024, T = 20) on 2 048 rollouts filled the way bench.py fills them: conv_1 of all
    21 504 frame stacks, its weight gradient over the 20 480 sequence rows and the 2592 -> 256 layer's forward passes
    (1 024 bootstrap rows, 20 480 sequence rows) of one eager fused step against fp64."""
    from distributed_rl_b200 import impala
    B, T, N = 1024, 20, 2048
    cfg = impala.ImpalaConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, UNROLL_STEP=T, LEARNER_DEVICE="cuda:0")
    torch.manual_seed(0)
    lrn = impala.Learner(cfg, start_replay=False)
    st = lrn._memory.store
    g = _gen(0xB208)
    st.fill_hash(N, seed=0xB204)
    st.field_view("action").copy_(torch.randint(0, 6, (N, T), device="cuda", generator=g, dtype=torch.int32))
    st.field_view("mu").copy_(torch.rand(N, T, device="cuda", generator=g) * 0.85 + 0.05)
    st.field_view("reward").copy_(torch.randn(N, T, device="cuda", generator=g))
    st.field_view("done").copy_((torch.rand(N, device="cuda", generator=g) > 0.05).float())
    st.build(torch.ones(N, device="cuda"))
    spies = _Spies(monkeypatch, R, L)
    lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    n = {k: len(v) for k, v in spies.calls.items()}
    assert n["conv1_fused"] == 1 and n["conv1_wgrad"] == 1 and n["linear3x"] == 3, n
    spies.check("IMPALA step", R)
    st.close()
