"""The kernels only the Ape-X learner step runs, against fp64 at bench.py's shapes (cfg/ape_x.json: B = 512, conv_3
output (B, 64, 7, 7) channels_last, the two first-layer heads [512][3136] stacked to N = 1024, Wa [6][512], Wv [1][512]).

A. The fused heads op (linear.relu_flat_heads_dueling: k_pack_act_nhwc's ReLU + NHWC -> NCHW flatten, the 3xTF32 GEMM
   left as K-split partials, b2rl_dueling_forward summing them), its backward (b2rl_unflatten_relu_mask summing dL/dy's
   partials, the joint dL/dW GEMM into adjacent .grad rows, the deferred b2rl_dueling_backward_w) and conv_1 over an
   Ape-X replay, on synthetic adversarial inputs.
B. Every hand-written kernel of one real eager Ape-X step with every default flag, on the inputs it actually received:
   conv_1 and its weight gradient, the batched and the target heads passes, the target kernel, the heads' backward,
   the gradients as the optimizer read them and the fused centered RMSprop of every tensor, then the resident operand
   images against a repack of the new weights.
C. The captured step against the eager one at B = 512, bit for bit, for 24 steps.

The bounds are the per-element fp64 bounds of tests/fp64_bounds.py; each checker prints its [err/tol] ratio."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fp64_bounds import (_gen, check_conv1, check_dueling_backward, check_gemm,  # noqa: E402
                         check_heads_dueling_forward, check_relu_flat_dgrad, check_rmsprop_centered, check_wgrad,
                         relu_flat)

B, C, HW, H, A = 512, 64, 49, 512, 6
K = C * HW
LOG2N = 14                       # 2^14 slots (0.9 GB): enough for B = 512 draws
# check_gemm's max-relative sanity ratio against cuBLAS fp32 for the Ape-X heads' GEMMs.  Measured on an H100 SXM
# (132 SMs, 700 W): the weight gradient [1024 x 512] x [3136 x 512]^T (one split of 16 chunks) errs 4.8e-6 of max|ref|,
# 11x cuBLAS fp32's 4.3e-7, and 4.1e-6 (5.8x) without the 1e4 activation; the real step's batched forward 5.8e-6,
# 9.7x.  The error follows the magnitude the fp32 accumulator holds: a 1e4 activation at the first contraction index
# puts the largest error in its own column, at the last index that column errs 20x less.  Every element stays inside
# check_gemm's derived bound (at most 0.3 of it), and TF32 / 20, the ratio a dropped lo term would break, holds with
# 60x to spare.
VS_CUBLAS = 16


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


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------- #
# A. the Ape-X-only kernels at the step's shapes, synthetic inputs              #
# --------------------------------------------------------------------------- #
def _heads_inputs(M, seed):
    """conv_3's output y (M, 64, 7, 7) channels_last: about half negative (the ReLU mask), channel 5 negative everywhere
    (a dead feature: 49 zero columns of the A operand) and one entry of 1e4; the two first-layer heads and the tail's
    weights."""
    g = _gen(seed)
    y = torch.randn(M, C, 7, 7, device="cuda", generator=g) * 0.5
    y[:, 5] = -y[:, 5].abs() - 0.01
    y[0, 0, 0, 0] = 1e4
    y = y.contiguous(memory_format=torch.channels_last)
    ws = [torch.empty(H, K, device="cuda").uniform_(-K ** -0.5, K ** -0.5, generator=g) for _ in range(2)]
    wa = torch.randn(A, H, device="cuda", generator=g) * 0.05
    wv = torch.randn(1, H, device="cuda", generator=g) * 0.05
    return y, ws, wa, wv


@pytest.mark.parametrize("M", [1024, 512, 300])
def test_relu_flat_heads_dueling_forward(L, M):
    """M = 1024: the batched online pass; 512: the target pass; 300: ragged.  With grad enabled (h is written; taken
    from an OutputTape) h is held to the 3xTF32 GEMM's bound against flatten_NCHW(relu(y)) @ cat(W)^T, q to the tail's
    bound plus h's own propagated through it; without grad (need_h false) q is the same bit for bit."""
    y, ws, wa, wv = _heads_inputs(M, 40 + M)
    with torch.enable_grad(), L.OutputTape.record() as tape:
        q = L.relu_flat_heads_dueling(y.requires_grad_(), [w.requires_grad_() for w in ws], wa, wv)
    h = tape.outs[0]
    assert len(tape.outs) == 2 and torch.equal(tape.outs[1], q.detach()) and h.shape == (M, 2 * H)
    with torch.no_grad():
        q_nh = L.relu_flat_heads_dueling(y, ws, wa, wv)
    assert torch.equal(q.detach(), q_nh)
    y = y.detach()
    ws = [w.detach() for w in ws]
    check_gemm(f"relu_flat_heads h M={M}", relu_flat(y).float(), torch.cat(ws, 0), h.detach())
    check_heads_dueling_forward(f"relu_flat_heads_dueling M={M}", y, ws, wa, wv, q_nh)


def _gq(M, seed):
    """dL/dQ of the Ape-X loss: each row one-hot at the taken action (-w td / B), about 10 % of the rows all zero (TD
    error clipped)."""
    g = _gen(seed)
    gq = torch.zeros(M, A, device="cuda")
    act = torch.randint(0, A, (M,), device="cuda", generator=g)
    val = torch.randn(M, device="cuda", generator=g) / M
    val *= torch.rand(M, device="cuda", generator=g) > 0.1
    gq[torch.arange(M, device="cuda"), act] = val
    return gq


class _BackwardSpy:
    """Record the inputs and the dL/dh of linear._dueling_backward during one backward pass."""

    def __init__(self, monkeypatch, L):
        self.calls = []
        orig = L._dueling_backward

        def spy(h, wa, wv, gq, need_gh, need_w):
            rec = dict(h=h.detach().clone(), wa=wa.detach().clone(), wv=wv.detach().clone(), gq=gq.detach().clone())
            res = orig(h, wa, wv, gq, need_gh, need_w)
            rec["gh"] = None if res[0] is None else res[0].detach().clone()
            self.calls.append(rec)
            return res
        monkeypatch.setattr(L, "_dueling_backward", spy)


@pytest.mark.parametrize("sink", [False, True])
def test_relu_flat_heads_dueling_backward(L, monkeypatch, sink):
    """Backward at M = 512 of the op, with Ape-X's dL/dQ: dL/dh, dL/dWa, dL/dWv against fp64 autograd of the tail;
    dL/dy (channels_last, zero wherever y <= 0) against fp64 per element; dL/dW of both heads against
    gh^T @ flatten_NCHW(relu(y)).  `sink`: inside an active WeightGradSink with grads_are_zero and the weights' .grad
    laid out by optim.flat_grads, so one GEMM writes both heads' dL/dW into their adjacent .grad rows and
    b2rl_dueling_backward_w runs deferred on the sink's lane."""
    from distributed_rl_b200.linear import WeightGradSink, _stacked_rows
    from distributed_rl_b200.optim import flat_grads
    y, ws, wa, wv = _heads_inputs(B, 50)
    y.requires_grad_()
    params = [w.requires_grad_() for w in ws] + [wa.requires_grad_(), wv.requires_grad_()]
    gq = _gq(B, 51)
    spy = _BackwardSpy(monkeypatch, L)
    if sink:
        flat = flat_grads(params)
        assert not flat.any() and _stacked_rows([w.grad for w in ws]) is not None
        sk = WeightGradSink("cuda:0")
        sk.grads_are_zero = True
        added = []
        orig_acc = sk.accumulate
        sk.accumulate = lambda p, g: (added.append(id(p)), orig_acc(p, g))[1]
        with sk.active():
            L.relu_flat_heads_dueling(y, ws, wa, wv).backward(gq)
        sk.join()
        assert not any(id(w) in added for w in ws), "the heads' dL/dW was not written by the joint GEMM"
        assert id(wa) in added and id(wv) in added
    else:
        L.relu_flat_heads_dueling(y, ws, wa, wv).backward(gq)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert len(spy.calls) == 1
    c = spy.calls[0]
    yd = y.detach()
    assert torch.equal(c["gq"], gq)
    what = f"heads backward sink={sink}"
    check_dueling_backward(what, c["h"], wa.detach(), wv.detach(), gq, c["gh"], wa.grad, wv.grad)
    assert y.grad.is_contiguous(memory_format=torch.channels_last)
    check_relu_flat_dgrad(what, yd, [w.detach() for w in ws], c["gh"], y.grad)
    check_gemm(f"{what} dL/dW", c["gh"].T.contiguous(), relu_flat(yd).float().T.contiguous(),
               torch.cat([w.grad for w in ws], 0), vs_cublas=VS_CUBLAS)


def _conv1_weights(seed):
    ws = [torch.empty(32, 4, 8, 8, device="cuda").uniform_(-0.0625, 0.0625, generator=_gen(seed + i)) for i in range(2)]
    ws[0][3] = 0.0                                   # an all-zero output channel
    ws[0][5, 0, 0, 0] = 0.9                          # one dominant weight: the small digits of the others matter
    return ws


def test_conv1_on_an_apex_replay(R):
    """conv_1 over a 2^14-slot Ape-X DeviceReplay (APEX_FIELDS, fill_hash): 512 draws with duplicates and slot 0, one
    slot's frames saturated.  The packs are built the way the learner builds them (one conv1_pack_jobs launch): online
    net alone over `state`, online + target over `next_state`, both with the ReLU; then the weight gradient over `state`
    masked by the ReLU output, added to a non-zero gradient."""
    N = 1 << LOG2N
    st = R.DeviceReplay(N, R.APEX_FIELDS, "cuda:0")
    try:
        st.fill_hash(N, seed=0xB205)
        st.field_view("state")[7] = 255
        st.field_view("next_state")[7] = 255
        idx = torch.randint(0, N, (B,), device="cuda", generator=_gen(60))
        idx[:4] = torch.tensor([0, 7, 7, 9])
        w_on, w_tg = _conv1_weights(61)
        pack1, pack2 = R.Conv1Pack(1, "cuda:0", 32), R.Conv1Pack(2, "cuda:0", 32)
        R.conv1_pack_jobs([(pack1, 0, w_on), (pack2, 0, w_on), (pack2, 1, w_tg)])
        s, ns = st.frame_source("state"), st.frame_source("next_state")
        y_s = R.conv1_fused(s, idx, pack1, relu=True)
        y_ns = R.conv1_fused(ns, idx, pack2, relu=True)
        check_conv1("conv1_fused Ape-X state, 1 net", s, idx, [w_on], y_s, True)
        check_conv1("conv1_fused Ape-X next_state, 2 nets", ns, idx, [w_on, w_tg], y_ns, True)
        assert (y_s[0][:, 3] == 0).all() and (y_ns[0][:, 3] == 0).all()
        g = _gen(62)
        gy = torch.randn(B, 32, 20, 20, device="cuda", generator=g)
        gy *= torch.logspace(-6, 0, B, device="cuda")[torch.randperm(B, device="cuda", generator=g)].view(B, 1, 1, 1)
        gy = gy.contiguous(memory_format=torch.channels_last)
        base = torch.randn(32, 4, 8, 8, device="cuda", generator=g) * 1e-3
        out = base.clone()
        R.conv1_wgrad(s, idx, gy, out=out, accumulate=True, relu_y=y_s[0])
        check_wgrad("conv1_wgrad Ape-X state", s, idx, gy, out, base=base, relu_y=y_s[0])
    finally:
        st.close()


# --------------------------------------------------------------------------- #
# B. one real Ape-X step at bench.py's shapes                                  #
# --------------------------------------------------------------------------- #
def _learner(cudnn_benchmark):
    """bench.py's Ape-X learner (every default flag) on 2^14 slots filled the way bench.py fills them, with a target
    network perturbed away from the online one (a swapped or stale operand image then changes the result)."""
    from distributed_rl_b200 import apex
    N = 1 << LOG2N
    cfg = apex.ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                          CUDNN_BENCHMARK=cudnn_benchmark)
    torch.manual_seed(0)
    lrn = apex.Learner(cfg, connect=None, start_replay=False)
    g = _gen(0xB209)
    with torch.no_grad():
        for p in lrn.target_model.parameters():
            p.add_(0.01 * torch.randn(p.shape, device="cuda", generator=g))
    st = lrn.memory.store
    st.fill_hash(N, seed=0xB200)
    g = _gen(0xB201)
    st.field_view("action").copy_(torch.randint(0, 6, (N,), device="cuda", generator=g, dtype=torch.int32))
    st.field_view("reward").copy_(torch.randn(N, device="cuda", generator=g).clamp_(-1, 1))
    st.field_view("done").copy_((torch.rand(N, device="cuda", generator=g) < 0.02).to(torch.uint8))
    st.build((torch.randn(N, device="cuda", generator=g).abs().clamp(max=1) + 1e-7) ** cfg.ALPHA)
    st.seed(1234, 0)
    return lrn


class _StepSpies:
    """Record what the hand-written kernels of an Ape-X step read and wrote.  Everything is cloned on the stream the
    call is issued on, so a clone sees exactly what the kernel launched next to it sees (or has just written)."""

    def __init__(self, monkeypatch, R, L):
        from distributed_rl_b200.optim import FusedRMSprop
        self.calls = {k: [] for k in ("conv1_fused", "conv1_wgrad", "heads", "dueling_backward", "relu_flat_backward",
                                      "apex_target", "launch")}
        self.packed = {}
        o_jobs, o_fused, o_wgrad, o_target = R.conv1_pack_jobs, R.conv1_fused, R.conv1_wgrad, R.apex_target
        o_heads, o_duel_bw, o_flat_bw = L.relu_flat_heads_dueling, L._dueling_backward, L._relu_flat_backward
        o_launch = FusedRMSprop._launch
        rec = self.calls

        def conv1_pack_jobs(jobs):
            for p, net, w in jobs:
                self.packed[(id(p), net)] = w.detach().float().clone()
            return o_jobs(jobs)

        def conv1_fused(frames, idx, pack, relu=False, out=None):
            res = o_fused(frames, idx, pack, relu=relu, out=out)
            rec["conv1_fused"].append(dict(frames=frames, idx=None if idx is None else idx.clone(), relu=relu,
                                           weights=[self.packed[(id(pack), i)] for i in range(pack.n_nets)],
                                           outs=[o.clone() for o in res]))
            return res

        def conv1_wgrad(frames, idx, gy, out=None, accumulate=False, relu_y=None):
            base = out.clone() if (out is not None and accumulate) else None
            res = o_wgrad(frames, idx, gy, out=out, accumulate=accumulate, relu_y=relu_y)
            rec["conv1_wgrad"].append(dict(frames=frames, idx=None if idx is None else idx.clone(),
                                           gy=gy.detach().clone(), base=base, got=res.detach().clone(),
                                           relu_y=None if relu_y is None else relu_y.detach().clone()))
            return res

        def heads(y, ws, wa, wv, cache=None):
            tape = L._TAPE
            mode = None if tape is None else tape.mode
            n0 = len(tape.outs) if mode == "record" else None
            grad = torch.is_grad_enabled()
            q = o_heads(y, ws, wa, wv, cache)
            rec["heads"].append(dict(y=y.detach().clone(), ws=[w.detach().clone() for w in ws],
                                     wa=wa.detach().clone(), wv=wv.detach().clone(), q=q.detach().clone(),
                                     h=tape.outs[n0].detach().clone() if mode == "record" else None,
                                     grad=grad, tape=mode))
            return q

        def dueling_backward(h, wa, wv, gq, need_gh, need_w):
            r = dict(h=h.detach().clone(), wa=wa.detach().clone(), wv=wv.detach().clone(), gq=gq.detach().clone())
            res = o_duel_bw(h, wa, wv, gq, need_gh, need_w)
            r["gh"] = None if res[0] is None else res[0].detach().clone()
            rec["dueling_backward"].append(r)
            return res

        def relu_flat_backward(y, ws, cache, gh, need_gy, need_gw):
            r = dict(y=y.detach().clone(), ws=[w.detach().clone() for w in ws], gh=gh.detach().clone())
            res = o_flat_bw(y, ws, cache, gh, need_gy, need_gw)
            r["gy"] = None if res[0] is None else res[0].detach().clone()
            rec["relu_flat_backward"].append(r)
            return res

        def apex_target(q_s, qn_online, qn_target, action, reward, notdone, weight, gamma_n, alpha, **kw):
            r = dict(q=q_s.clone(), qo=qn_online.clone(), qt=qn_target.clone(), a=action.clone(), r=reward.clone(),
                     nd=notdone.clone(), w=weight.clone(), gamma_n=gamma_n, alpha=alpha)
            res = o_target(q_s, qn_online, qn_target, action, reward, notdone, weight, gamma_n, alpha, **kw)
            r["out"] = {k: None if v is None else v.clone() for k, v in res.items()}
            rec["apex_target"].append(r)
            return res

        def launch(opt, lo, hi, norm_out):
            def state(i, p):
                return dict(p=p.detach().clone(), g=p.grad.clone(), sq=opt.square_avg[i].clone(),
                            ga=opt.grad_avg[i].clone())
            pre = [state(i, p) for i, p in enumerate(opt.params[lo:hi], lo)]
            o_launch(opt, lo, hi, norm_out)
            post = [state(i, p) for i, p in enumerate(opt.params[lo:hi], lo)]
            rec["launch"].append(dict(lo=lo, hi=hi, pre=pre, post=post))

        monkeypatch.setattr(R, "conv1_pack_jobs", conv1_pack_jobs)
        monkeypatch.setattr(R, "conv1_fused", conv1_fused)
        monkeypatch.setattr(R, "conv1_wgrad", conv1_wgrad)
        monkeypatch.setattr(R, "apex_target", apex_target)
        monkeypatch.setattr(L, "relu_flat_heads_dueling", heads)
        monkeypatch.setattr(L, "_dueling_backward", dueling_backward)
        monkeypatch.setattr(L, "_relu_flat_backward", relu_flat_backward)
        monkeypatch.setattr(FusedRMSprop, "_launch", launch)

    def clear(self):
        for v in self.calls.values():
            v.clear()


def _heads_params(model):
    """(first-layer weights [adv, val], Wa, Wv) of the dueling heads, in operand order."""
    group, ws = model.head_pieces()[0]
    duel = model._dueling[group]
    return ws, getattr(model, duel["adv"]).MLP_2.weight, getattr(model, duel["val"]).MLP_2.weight


def test_one_apex_step_every_kernel_against_fp64(R, L, monkeypatch):
    """bench.py's Ape-X line (B = 512, every default flag: batched online pass, parallel forwards, deferred weight
    gradients, early heads update, fused optimizer, resident operand images) on 2^14 slots, with bench.py's library
    knobs (cuDNN autotune, TF32 convolutions: every check is made on the inputs a kernel actually received, so cuDNN's
    precision enters no bound).  Two eager steps move the optimizer state and the online images; the third is checked
    kernel by kernel against fp64."""
    from test_gpu_15_resident_images import _assert_images_current
    torch.backends.cudnn.benchmark = True              # bench.py's library knobs (the conftest fixture restores them)
    torch.backends.cudnn.deterministic = False
    torch.backends.cudnn.allow_tf32 = True
    lrn = _learner(cudnn_benchmark=True)
    st = lrn.memory.store
    spies = _StepSpies(monkeypatch, R, L)
    for _ in range(2):
        lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    spies.clear()
    out = lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    calls = spies.calls
    n = {k: len(v) for k, v in calls.items()}
    assert n == {"conv1_fused": 2, "conv1_wgrad": 1, "heads": 3, "dueling_backward": 1, "relu_flat_backward": 1,
                 "apex_target": 1, "launch": 2}, n
    assert lrn._fused.resident is not None and lrn._fused.sink is not None and lrn._fused.early_ok

    # conv_1: online over s, online + target over s'; its weight gradient added to .grad
    for c in calls["conv1_fused"]:
        check_conv1(f"Ape-X step conv1_fused {len(c['weights'])} net(s)", c["frames"], c["idx"], c["weights"],
                    c["outs"], c["relu"])
    c = calls["conv1_wgrad"][0]
    assert c["base"] is not None and c["relu_y"] is not None
    check_wgrad("Ape-X step conv1_wgrad", c["frames"], c["idx"], c["gy"], c["got"], base=c["base"], relu_y=c["relu_y"])

    # heads forward: the batched online pass (M = 1024, recorded), the target pass (M = 512), the s half replayed
    target, batched, replayed = calls["heads"]                 # issue order: the target pass forks first
    assert (target["tape"], batched["tape"], replayed["tape"]) == (None, "record", "replay")
    assert batched["y"].shape[0] == 2 * B and target["y"].shape[0] == B and replayed["grad"]
    ws_on, wa_on, wv_on = _heads_params(lrn.model)
    ws_tg, wa_tg, wv_tg = _heads_params(lrn.target_model)
    check_gemm("Ape-X step batched pass h", relu_flat(batched["y"]).float(), torch.cat(batched["ws"], 0), batched["h"],
               vs_cublas=VS_CUBLAS)
    for what, c in (("batched pass", batched), ("target pass", target)):
        check_heads_dueling_forward(f"Ape-X step {what}", c["y"], c["ws"], c["wa"], c["wv"], c["q"])
    assert all(torch.equal(a, b) for a, b in zip(target["ws"] + [target["wa"], target["wv"]], ws_tg + [wa_tg, wv_tg]))
    assert not torch.equal(batched["ws"][0], target["ws"][0]) and not torch.equal(batched["wa"], target["wa"])
    assert torch.equal(replayed["q"], batched["q"][:B])
    assert torch.equal(replayed["y"], batched["y"][:B])

    # target kernel on its own inputs against the numpy oracle
    from oracle import oracle as O
    t = calls["apex_target"][0]
    np_in = {k: t[k].cpu().numpy() for k in ("q", "qo", "qt", "a", "r", "nd", "w")}
    assert torch.equal(t["q"], batched["q"][:B]) and torch.equal(t["qo"], batched["q"][B:])
    assert torch.equal(t["qt"], target["q"])
    tgt, td, prio, gq, _ = O.apex_target(np_in["q"], np_in["qo"], np_in["qt"], np_in["a"], np_in["r"], np_in["nd"],
                                         np_in["w"], t["gamma_n"], t["alpha"])
    np.testing.assert_array_equal(t["out"]["td"].cpu().numpy(), td)
    np.testing.assert_array_equal(t["out"]["grad_q"].cpu().numpy(), gq)
    np.testing.assert_allclose(t["out"]["target"].cpu().numpy(), tgt, rtol=0, atol=1e-5)
    np.testing.assert_allclose(t["out"]["prio"].cpu().numpy(), prio, rtol=2.4e-7)

    # heads backward: the tail's dL/dh and the flatten + ReLU mask's dL/dy
    db, fb = calls["dueling_backward"][0], calls["relu_flat_backward"][0]
    assert torch.equal(db["h"], batched["h"][:B]) and torch.equal(db["gq"], t["out"]["grad_q"])
    assert torch.equal(fb["gh"], db["gh"]) and torch.equal(fb["y"], batched["y"][:B])
    check_relu_flat_dgrad("Ape-X step", fb["y"], fb["ws"], fb["gh"], fb["gy"])

    # the gradients as the optimizer read them (the early heads update on the sink's lane, the rest after backward)
    opt = lrn.optim
    pre, post = {}, {}
    for c in calls["launch"]:
        for i, (a, b) in enumerate(zip(c["pre"], c["post"]), c["lo"]):
            assert i not in pre, f"tensor {i} stepped twice"
            pre[i], post[i] = a, b
    assert sorted(pre) == list(range(len(opt.params)))
    at = {id(p): i for i, p in enumerate(opt.params)}
    early = next(c for c in calls["launch"] if c["lo"] == at[id(ws_on[0])])
    assert {at[id(p)] for p in (*ws_on, wa_on, wv_on)} == set(range(early["lo"], early["hi"])), "the heads' early update"
    g_ws = torch.cat([pre[at[id(w)]]["g"] for w in ws_on], 0)
    check_gemm("Ape-X step heads dL/dW as read by the optimizer", db["gh"].T.contiguous(),
               relu_flat(fb["y"]).float().T.contiguous(), g_ws, vs_cublas=VS_CUBLAS)
    check_dueling_backward("Ape-X step (dL/dWa, dL/dWv as read by the optimizer)", db["h"], db["wa"], db["wv"], db["gq"],
                           db["gh"], pre[at[id(wa_on)]]["g"], pre[at[id(wv_on)]]["g"])

    # the fused centered RMSprop of every tensor (heads: the 32x32 tile path writing the images; the rest: plain)
    info = lrn.cfg.OPTIM_INFO
    names = {id(p): nm for nm, p in lrn.model.named_parameters()}
    for i, p in enumerate(opt.params):
        check_rmsprop_centered(f"Ape-X step RMSprop {names[id(p)]}", pre[i], post[i], info["lr"], info["alpha"],
                               info["eps"])
    norm = sum(pre[i]["g"].double().norm() for i in pre).sqrt().item()
    got = out["p_norm"].item()
    print(f"[err/tol] Ape-X step p_norm: {abs(got - norm) / (1e-6 * norm):.3g}")
    assert abs(got - norm) <= 1e-6 * norm, (got, norm)

    # the resident images are the packs of the new weights, bit for bit
    _assert_images_current(lrn.model, True)
    _assert_images_current(lrn.target_model, False)
    st.close()


# --------------------------------------------------------------------------- #
# C. the captured step equals the eager step at B = 512                        #
# --------------------------------------------------------------------------- #
def _state(lrn, out):
    st = lrn.memory.store
    return dict(idx=out["idx"].clone(), w=lrn._cur["w"].clone(), prio=out["prio"].clone(),
                scalars=out["scalars"].clone(), p_norm=out["p_norm"].clone(),
                params=[p.detach().clone() for p in lrn.model.parameters()],
                sq=[t.clone() for t in lrn.optim.square_avg], ga=[t.clone() for t in lrn.optim.grad_avg],
                leaves=st.priorities(), root=st.stats(lrn.cfg.BETA))


def test_captured_step_equals_the_eager_step_at_b512():
    """Two identical learners (part B's configuration, cuDNN heuristics and deterministic algorithms): one builds its
    graph (3 eager warm-ups, the capture, one replay: 4 bodies) and replays it 20 times, the other runs 4 + 20 eager
    steps.  After each: draws, IS weights, priorities, the step's scalars, every parameter, both optimizer states and
    the tree's leaves and root bit for bit; the gradient norm (fp64 atomics, order-dependent at 1e-16) to 1e-6."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if torch.cuda.mem_get_info()[0] < 20 << 30:
        pytest.skip("needs about 16 GB of free device memory")
    graph, eager = _learner(cudnn_benchmark=False), _learner(cudnn_benchmark=False)
    for step in range(21):
        a = _state(graph, graph.fused_step(use_graph=True))
        for _ in range(4 if step == 0 else 1):
            o = eager.fused_step(use_graph=False)
        b = _state(eager, o)
        torch.cuda.synchronize()
        for k in ("idx", "w", "prio", "scalars", "leaves", "root"):
            assert torch.equal(a[k], b[k]), (step, k)
        for k in ("params", "sq", "ga"):
            for i, (x, y) in enumerate(zip(a[k], b[k])):
                assert torch.equal(x, y), (step, k, i)
        assert abs(a["p_norm"].item() - b["p_norm"].item()) <= 1e-6 * abs(b["p_norm"].item()), step
    assert graph._graph is not None and eager._graph is None
    graph.memory.store.close()
    eager.memory.store.close()
