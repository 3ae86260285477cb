"""conv_1 (forward and weight gradient), the 3xTF32 dense layers and the dueling tail against fp64 at the shapes the
R2D2 (B = 64, T = 80, MEM = 20) and IMPALA (B = 1024, T = 20) learner steps run them, first on synthetic inputs, then on
the inputs of one real eager step of each learner.

Every output element is held to its own bound, computed by the same fp64 reference applied to absolute values
(`mag`), so the bound grows with the length of the sum behind that element; u = 2^-24.  The bound of each kernel is
written in its checker's docstring (tests/fp64_bounds.py).  The fp64 references run on the device, a chunk of frame
stacks at a time; the frames are drawn on the device from seeded generators."""
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fp64_bounds import (_frames, _gen, check_conv1, check_dueling_backward, check_dueling_forward,  # noqa: E402
                         check_gemm, check_wgrad)

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


def r2d2_learner(N=256, payload_pool=0):
    """bench.py's R2D2 learner (B = 64, T = 80, MEM = 20) with N sum-tree slots, filled the way bench.py fills it:
    hashed frames, seeded small fields and priorities.  payload_pool > 0: bench.py's row map, N slots over that many
    stored sequences (slot s reads row s % payload_pool)."""
    from distributed_rl_b200 import r2d2
    B, T = 64, 80
    P = payload_pool or N
    cfg = r2d2.R2D2Config(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, PAYLOAD_POOL=payload_pool,
                          FIXED_TRAJECTORY=T, MEM=20, LEARNER_DEVICE="cuda:0")
    torch.manual_seed(0)
    lrn = r2d2.Learner(cfg, start_replay=False)
    st, pool = lrn.memory.store, lrn.memory.pool
    g = _gen(0xB207)
    pool.fill_hash(P, seed=0xB203)
    pool.field_view("action").copy_(torch.randint(0, 6, (P, T), device="cuda", generator=g, dtype=torch.int32))
    pool.field_view("reward").copy_(torch.randn(P, T, device="cuda", generator=g))
    pool.field_view("h0").copy_(torch.randn(P, 512, device="cuda", generator=g) * 0.1)
    pool.field_view("h1").copy_(torch.randn(P, 512, device="cuda", generator=g) * 0.1)
    pool.field_view("notdone").copy_((torch.rand(P, device="cuda", generator=g) > 0.02).float())
    st.build((torch.randn(N, device="cuda", generator=g).abs().clamp(max=1) + 1e-7) ** cfg.ALPHA)
    st.seed(1234, 0)
    return lrn


def impala_learner():
    """bench.py's IMPALA learner (B = 1024, T = 20) on 2 048 rollouts filled the way bench.py fills them."""
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
    return lrn


def test_one_r2d2_step_at_the_bench_shapes(R, L, monkeypatch):
    """bench.py's R2D2 line (B = 64, T = 80, MEM = 20) on a 256-sequence replay filled the way bench.py fills it: every
    conv_1, conv_1 weight gradient, heads GEMM and dueling tail of one eager fused step against fp64."""
    lrn = r2d2_learner()
    st = lrn.memory.store
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
    lrn = impala_learner()
    st = lrn._memory.store
    spies = _Spies(monkeypatch, R, L)
    lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    n = {k: len(v) for k, v in spies.calls.items()}
    assert n["conv1_fused"] == 1 and n["conv1_wgrad"] == 1 and n["linear3x"] == 3, n
    spies.check("IMPALA step", R)
    st.close()
