"""The R2D2 (B = 64, T = 80, MEM = 20, bench.py's 2^20 slots over a 256-sequence payload pool) and IMPALA (B = 1024,
T = 20) learner steps against fp64 at bench.py's shapes.

A. The kernels test_gpu_22_step_shapes does not reach, on the inputs one real eager step gave them: the heads'
   3xTF32 dL/dx and dL/dW, R2D2's dueling-tail backward and target kernel, IMPALA's V-trace.
B. The whole eager step against a restatement of it without the library, in fp64, fp32 and TF32 (plain GraphAgent
   forward, cuDNN / cuBLAS only), held to check_vs_reference; two negative controls wire a fault into the step and
   must fail the same comparison.
C. b2rl_vtrace and b2rl_r2d2_target at their edges.

The bounds are those of tests/fp64_bounds.py; each checker prints its [err/tol] or [err/ref] ratio."""
import contextlib
import copy

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fp64_bounds import (check_dueling_backward, check_gemm, check_vs_reference, check_vtrace,  # noqa: E402
                         vtrace_inputs)
from test_gpu_22_step_shapes import _Spies, impala_learner, r2d2_learner  # noqa: E402

SLOTS, POOL = 2 ** 20, 256           # bench.py's R2D2 row map: slot s reads payload row s % POOL
# check_gemm's max-relative sanity ratio against cuBLAS fp32 for R2D2's heads dL/dx on the step's own inputs.  Measured
# on an H100 SXM (700 W): 3xTF32 4.4e-6 of max|ref|, cuBLAS fp32 4.6e-7: 9.5x, above the 8x test_gpu_22 measured on
# synthetic inputs (cuBLAS fp32 picks a more accurate kernel for this shape, see there).  Every element stays within
# 0.05 of check_gemm's derived bound and TF32 / 20 holds with 3.4x to spare; 16 is test_gpu_25's VS_CUBLAS.
VS_CUBLAS_DX = 16


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    free, _ = torch.cuda.mem_get_info()
    if free < 40 << 30:
        pytest.skip(f"needs about 40 GB of free device memory, {free / 2 ** 30:.1f} GB free")
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


def _clone(x):
    return x.detach().clone() if torch.is_tensor(x) else x


class _StepSpies(_Spies):
    """test_gpu_22's spies plus the rest of one step: the draw (`draw_owner.draw_name`), the heads' backward
    (_Linear3x.backward), the dueling tail's backward, the target kernel (replay.r2d2_target or replay.vtrace), the
    gradient every Tensor.backward call is given, and every parameter's .grad as the learner's `step` receives it
    (cloned before the clip)."""

    def __init__(self, monkeypatch, R, L, lrn, draw_owner, draw_name):
        super().__init__(monkeypatch, R, L)
        self.calls.update(draw=[], linear3x_backward=[], dueling_backward=[], r2d2_target=[], vtrace=[], backward=[])
        self.grads = None
        orig_draw = getattr(draw_owner, draw_name)
        orig_lin_bwd, orig_duel_bwd = L._Linear3x.backward, L._dueling_backward
        orig_target, orig_vtrace = R.r2d2_target, R.vtrace
        orig_tensor_bwd, orig_step = torch.Tensor.backward, lrn.step

        def draw(*a, **k):
            res = orig_draw(*a, **k)
            self.calls["draw"].append(tuple(_clone(t) for t in res) if isinstance(res, tuple) else _clone(res))
            return res

        def lin_backward(ctx, gy):
            x, *ws = ctx.saved_tensors
            res = orig_lin_bwd(ctx, gy)
            self.calls["linear3x_backward"].append(dict(
                x=_clone(x), w=torch.cat([w.detach() for w in ws], 0), gy=gy.detach().contiguous().clone(),
                gx=_clone(res[0]), gw=None if res[2] is None else torch.cat([g.detach() for g in res[2:]], 0)))
            return res

        def dueling_backward(h, wa, wv, gq, need_gh, need_w):
            res = orig_duel_bwd(h, wa, wv, gq, need_gh, need_w)
            self.calls["dueling_backward"].append(dict(h=_clone(h), wa=_clone(wa), wv=_clone(wv), gq=_clone(gq),
                                                       gh=_clone(res[0]), gwa=_clone(res[1]), gwv=_clone(res[2])))
            return res

        def r2d2_target(*a, **k):
            out = orig_target(*a, **k)
            self.calls["r2d2_target"].append(dict(args=[_clone(t) for t in a], kw=dict(k), out=out,
                                                  got={n: _clone(t) for n, t in out.items()}))
            return out

        def vtrace(*a):
            vt, adv = orig_vtrace(*a)
            self.calls["vtrace"].append(dict(args=[_clone(t) for t in a], vt=_clone(vt), adv=_clone(adv)))
            return vt, adv

        def tensor_backward(t, gradient=None, *a, **k):
            self.calls["backward"].append(gradient)
            return orig_tensor_bwd(t, gradient, *a, **k)

        def step(*a, **k):
            self.grads = {n: _clone(p.grad) for n, p in lrn.model.named_parameters()}
            return orig_step(*a, **k)

        self.masks = {}                 # ReLU module name -> (input > 0) of the learner's pass with grad
        self.hooks = []
        for name, mod in lrn.model.named_modules():
            if isinstance(mod, torch.nn.ReLU):
                def relu_hook(m, inp, out, name=name):
                    if torch.is_grad_enabled():
                        self.masks[name] = inp[0].detach() > 0
                self.hooks.append(mod.register_forward_hook(relu_hook))

        monkeypatch.setattr(draw_owner, draw_name, draw)
        monkeypatch.setattr(L._Linear3x, "backward", staticmethod(lin_backward))
        monkeypatch.setattr(L, "_dueling_backward", dueling_backward)
        monkeypatch.setattr(R, "r2d2_target", r2d2_target)
        monkeypatch.setattr(R, "vtrace", vtrace)
        monkeypatch.setattr(torch.Tensor, "backward", tensor_backward)
        monkeypatch.setattr(lrn, "step", step)


    def remove_hooks(self):
        for h in self.hooks:
            h.remove()


def _r2d2_step(R, L, monkeypatch, fault=None):
    """One eager R2D2 step at bench.py's shapes and row map -> (learner, snapshots of the online and target nets
    before it, spies, fused_step's result).  `fault(monkeypatch, learner)` wires a fault in after the spies."""
    lrn = r2d2_learner(SLOTS, POOL)
    snap = [copy.deepcopy(m) for m in (lrn.model, lrn.target_model)]
    spies = _StepSpies(monkeypatch, R, L, lrn, lrn.memory.store, "sample")
    if fault is not None:
        fault(monkeypatch, lrn)
    res = lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    spies.remove_hooks()
    adv, val = _dueling_names(lrn.model)        # the fused dueling tail's ReLU: its input h, advantage | value
    h = spies.calls["dueling_backward"][0]["h"]
    H = h.shape[1] // 2
    spies.masks.update({f"{adv}.act_1": h[:, :H] > 0, f"{val}.act_1": h[:, H:] > 0})
    return lrn, snap, spies, res


def _impala_step(R, L, monkeypatch, fault=None):
    """One eager IMPALA step at bench.py's shapes -> (learner, snapshot of the net before it, spies)."""
    lrn = impala_learner()
    snap = copy.deepcopy(lrn.model)
    spies = _StepSpies(monkeypatch, R, L, lrn, lrn._memory, "draw")
    if fault is not None:
        fault(monkeypatch, lrn)
    lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    spies.remove_hooks()
    return lrn, snap, spies


def _close(lrn):
    mem = lrn.memory
    for st in {id(s): s for s in (mem.store, getattr(mem, "pool", mem.store))}.values():
        st.close()


def _dueling_names(model):
    d = next(iter(model._dueling.values()))
    return d["adv"], d["val"]


# --------------------------------------------------------------------------- #
# A. the remaining kernels of one eager step, on the inputs they received      #
# --------------------------------------------------------------------------- #
def test_r2d2_step_kernels_on_their_inputs(R, L, monkeypatch):
    """Every conv_1, heads GEMM and dueling forward of the step (test_gpu_22's checks, here through the 2^20-slot row
    map), the heads' dL/dx ([3840 x 1024] . [1024 x 512], held to VS_CUBLAS_DX x cuBLAS fp32) and dL/dW
    (contraction over M = 3840), the dueling tail's backward, and the target kernel bit for bit against the oracle.
    The gradients `step` sees on the heads' first and second layers are the ones these kernels returned: no other
    term reaches them.  The grad_q that q.backward receives is the tensor the target kernel wrote."""
    lrn, _, spies, _ = _r2d2_step(R, L, monkeypatch)
    c = spies.calls
    n = {k: len(c[k]) for k in ("conv1_fused", "conv1_wgrad", "linear3x_backward", "dueling_backward",
                                "r2d2_target", "backward")}
    assert n == dict(conv1_fused=2, conv1_wgrad=1, linear3x_backward=1, dueling_backward=1, r2d2_target=1,
                     backward=1), n
    spies.check("R2D2 step", R)
    adv, val = _dueling_names(lrn.model)

    b = c["linear3x_backward"][0]
    assert b["x"].shape == (3840, 512) and b["w"].shape == (1024, 512)
    check_gemm("R2D2 step heads dL/dx", b["gy"], b["w"].T.contiguous(), b["gx"], vs_cublas=VS_CUBLAS_DX)
    check_gemm("R2D2 step heads dL/dW", b["gy"].T.contiguous(), b["x"].T.contiguous(), b["gw"])
    g = spies.grads
    assert torch.equal(torch.cat([g[f"{adv}.MLP_1.weight"], g[f"{val}.MLP_1.weight"]], 0), b["gw"])

    d = c["dueling_backward"][0]
    check_dueling_backward("R2D2 step dueling_tail", d["h"], d["wa"], d["wv"], d["gq"], d["gh"], d["gwa"], d["gwv"])
    assert torch.equal(g[f"{adv}.MLP_2.weight"], d["gwa"]) and torch.equal(g[f"{val}.MLP_2.weight"], d["gwv"])

    t = c["r2d2_target"][0]
    q, qt, act, rew, nd, w, n_step, gamma, alpha, rescale = t["args"]
    assert q.shape == (60, 64, 6) and n_step == lrn.cfg.UNROLL_STEP
    tgt, td, prio, gq, info = O.r2d2_target(*(x.cpu().numpy() for x in (q, qt, act, rew, nd, w)), n_step, gamma,
                                            alpha, rescale)
    got = {k: v.cpu().numpy() for k, v in t["got"].items()}
    for name, ref in (("target", tgt), ("td", td), ("grad_q", gq)):
        assert np.array_equal(got[name].view(np.uint32), ref.view(np.uint32)), f"r2d2_target {name} differs"
    np.testing.assert_allclose(got["prio"], prio, rtol=5e-7)
    np.testing.assert_allclose(got["scalars"], [info["loss"], info["mean_value"]], rtol=2e-6, atol=1e-7)
    fed = c["backward"][0]
    assert fed is t["out"]["grad_q"] and torch.equal(fed, t["got"]["grad_q"])
    _close(lrn)


def test_impala_step_kernels_on_their_inputs(R, L, monkeypatch):
    """The 2592 -> 256 layer's dL/dx ([20480 x 256] . [256 x 2592]) and dL/dW (contraction over M = 20 480), and
    V-trace on the step's own inputs, against check_vtrace's fp64 bound and against oracle.vtrace at test_gpu_00's
    tolerance.  The gradient `step` sees on that layer is the one the GEMM returned."""
    lrn, _, spies = _impala_step(R, L, monkeypatch)
    c = spies.calls
    assert len(c["linear3x_backward"]) == 1 and len(c["vtrace"]) == 1, {k: len(v) for k, v in c.items()}
    b = c["linear3x_backward"][0]
    assert b["x"].shape == (20480, 2592) and b["w"].shape == (256, 2592)
    check_gemm("IMPALA step dense dL/dx", b["gy"], b["w"].T.contiguous(), b["gx"])
    check_gemm("IMPALA step dense dL/dW", b["gy"].T.contiguous(), b["x"].T.contiguous(), b["gw"])
    assert torch.equal(spies.grads["module01.MLP_1.weight"], b["gw"])

    v = c["vtrace"][0]
    pi, mu, value, boot, rew, gamma, lam, cbar, pbar = v["args"]
    assert pi.shape == (20, 1024)
    check_vtrace("IMPALA step vtrace", pi, mu, value, boot, rew, gamma, lam, cbar, pbar, v["vt"], v["adv"])
    ovt, oadv, _ = O.vtrace(*(x.cpu().numpy() for x in (pi, mu, value, boot, rew)), gamma, lam, cbar, pbar)
    np.testing.assert_allclose(v["vt"].cpu().numpy(), ovt, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(v["adv"].cpu().numpy(), oadv, rtol=1e-5, atol=1e-5)
    _close(lrn)


# --------------------------------------------------------------------------- #
# B. the whole step against an fp64 restatement                                #
# --------------------------------------------------------------------------- #
ARMS = (("fp64", torch.float64, False), ("fp32", torch.float32, False), ("tf32", torch.float32, True))


@contextlib.contextmanager
def _tf32(on):
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = on
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _plain(model, dtype):
    """A copy of `model` in `dtype` on the plain GraphAgent path: nn.Linear, cuDNN convolutions and LSTM, the
    dueling nodes one by one."""
    m = copy.deepcopy(model).to(dtype)
    m.dense_3xtf32 = m.fused_dueling_tail = m.fuse_sibling_heads = m.fused_relu_flatten = False
    return m


def _learner_masks(model, masks):
    """Make every ReLU of `model`'s pass with grad apply the learner's decision (the recorded input > 0) instead of
    its own: input * mask.  The arms take the learner's ReLU decisions as the learner's target kernel takes its own
    argmax: an activation within rounding of zero flips between precisions, and one flip moves a whole rank-1 term of
    the weight gradient behind it (1.5 % of max |dL/dW| of R2D2's first heads layer, measured without this split),
    so the comparison would measure which activations sit at zero rather than the arithmetic.  The forward values
    move by at most that activation's own tiny magnitude."""
    names = {n for n, m in model.named_modules() if isinstance(m, torch.nn.ReLU)}
    assert names == set(masks), (sorted(names), sorted(masks))
    for name, mod in model.named_modules():
        if name in masks:
            def hook(m, inp, out, mask=masks[name]):
                if torch.is_grad_enabled():
                    return inp[0] * mask.to(inp[0].dtype)
            mod.register_forward_hook(hook)
    return model


def _arms(restate):
    """restate(dtype) under each arm's TF32 setting -> {arm: result}; no libb2rl launch in any of them."""
    from distributed_rl_b200 import _lib
    n0 = _lib.load().b2rl_launch_count()
    out = {}
    for name, dtype, tf32 in ARMS:
        with _tf32(tf32):
            out[name] = restate(dtype)
    torch.cuda.synchronize()
    assert _lib.load().b2rl_launch_count() == n0, "the reference arms launched a libb2rl kernel"
    return out


class _Comparison:
    """check_vs_reference over every compared tensor of one step; the failures are collected and reported together."""

    def __init__(self, what, arms):
        self.what, self.arms, self.failed = what, arms, []

    def __call__(self, key, got, ref=lambda arm, key: arm[key], k=16, sharp=True):
        try:
            check_vs_reference(f"{self.what} {key}", got, *(ref(self.arms[a], key) for a in ("fp64", "fp32", "tf32")),
                               k=k, sharp=sharp)
        except AssertionError as e:
            self.failed.append(str(e))

    def grads(self, grads, k=None):
        """Every parameter's gradient; `k`: {parameter name: k} where it is not 16."""
        for name, g in grads.items():
            self(f"dL/d {name}", g, lambda arm, key: arm["grads"][key[5:]], k=(k or {}).get(name, 16))

    def check(self):
        assert not self.failed, "\n".join(self.failed)


def _r2d2_compare(lrn, snap, spies, res):
    """The R2D2 step's q, q_target, pre-clip gradients and p_norm against the restatement: the sequences read from the
    payload pool at idx % POOL, time-major by permute, burn-in without grad on both nets, then the window; the target
    kernel's own grad_q backpropagated through each arm's window q."""
    c, cfg = spies.calls, lrn.cfg
    T, MEM, B, A = cfg.FIXED_TRAJECTORY, cfg.MEM, cfg.BATCHSIZE, cfg.ACTION_SIZE
    idx, _, w = c["draw"][0]
    rows = idx % POOL
    assert torch.equal(rows, lrn.memory.rows_of(idx))
    pool = lrn.memory.pool
    f = {k: pool.field_view(k)[rows] for k in ("state", "action", "reward", "h0", "h1", "notdone")}
    q, qt, act, rew, nd, wt = c["r2d2_target"][0]["args"][:6]
    assert torch.equal(act, f["action"].long().t()[MEM:-1]) and torch.equal(rew, f["reward"].t()[MEM:-1])
    assert torch.equal(nd, f["notdone"]) and torch.equal(wt, w)
    grad_q = c["r2d2_target"][0]["got"]["grad_q"]
    frames = f["state"].permute(1, 0, 2, 3, 4)                  # (T, B, 4, 84, 84): time-major

    def restate(dtype):
        on, tg = _learner_masks(_plain(snap[0], dtype), spies.masks), _plain(snap[1], dtype)
        x = frames.to(dtype) / 255.0
        burn, window = x[:MEM].reshape(-1, 4, 84, 84), x[MEM:].reshape(-1, 4, 84, 84)
        hc = (f["h0"].to(dtype)[None], f["h1"].to(dtype)[None])
        for m in (on, tg):
            m.setCellState(hc)
        with torch.no_grad():
            for m in (on, tg):
                m.forward([burn, torch.tensor([MEM, B, -1])])
                m.detachCellState()
        shape = torch.tensor([T - MEM, B, -1])
        qa = on.forward([window, shape])[0].view(T - MEM, B, A)
        with torch.no_grad():
            qta = tg.forward([window, shape])[0].view(T - MEM, B, A)
        qa.backward(grad_q.to(dtype))
        grads = {n: p.grad for n, p in on.named_parameters()}
        return dict(q=qa.detach(), q_target=qta, grads=grads,
                    p_norm=torch.stack([g.norm() for g in grads.values()]).sum().sqrt())

    cmp = _Comparison("R2D2", _arms(restate))
    cmp("q", q)
    cmp("q_target", qt)
    cmp.grads(spies.grads)
    cmp("p_norm", res["p_norm"])
    cmp.check()


def _impala_compare(lrn, snap, spies):
    """The IMPALA step's pi_a, value, boot, objActor, criticLoss and pre-clip gradients against the restatement: the
    rollouts read from the store at the drawn slots, time-major by permute, the bootstrap stacks, then the sequence
    stacks; softmax and gather; the actor, entropy and critic loss formed from the learner's own vt and adv."""
    c, cfg = spies.calls, lrn.cfg
    T, B, A = cfg.UNROLL_STEP, cfg.BATCHSIZE, cfg.ACTION_SIZE
    idx = c["draw"][0]
    st = lrn._memory.store
    f = {k: st.field_view(k)[idx] for k in ("state", "action", "mu", "reward", "done")}
    pi, mu, value, boot, rew = c["vtrace"][0]["args"][:5]
    vt, adv = c["vtrace"][0]["vt"], c["vtrace"][0]["adv"]
    assert torch.equal(mu, f["mu"].t()) and torch.equal(rew, f["reward"].t())
    action = f["action"].long().t().reshape(-1, 1)              # time-major
    frames = f["state"].view(B, T + 1, 4, 84, 84).permute(1, 0, 2, 3, 4).contiguous()

    def restate(dtype):
        m = _learner_masks(_plain(snap, dtype), spies.masks)
        with torch.no_grad():
            out_last = m.forward([frames[T].to(dtype) / 255.0])[0]
        out = m.forward([frames[:T].reshape(-1, 4, 84, 84).to(dtype) / 255.0])[0]
        logits = out[:, :A]
        logp = torch.log_softmax(logits, dim=-1)
        entropy = -(logp.exp() * logp).sum(-1, keepdim=True)
        obj = torch.mean(logp.gather(1, action) * adv.to(dtype).view(-1, 1) + cfg.ENTROPY_R * entropy)
        critic = torch.mean((out[:, -1] - vt.to(dtype).view(-1)).pow(2)) / 2
        (-obj + critic).backward()
        return dict(pi_a=torch.softmax(logits.detach(), dim=-1).gather(1, action)[:, 0].view(T, B),
                    value=out[:, -1].detach().view(T, B), boot=out_last[:, -1] * f["done"].to(dtype),
                    objActor=obj.detach(), criticLoss=critic.detach(),
                    grads={n: p.grad for n, p in m.named_parameters()})

    cmp = _Comparison("IMPALA", _arms(restate))
    for key, got in (("pi_a", pi), ("value", value), ("boot", boot)):
        cmp(key, got)
    # The two losses are means over 20 480 terms, in which TF32's roundings average out: measured on an H100 SXM
    # (700 W), the TF32 arm errs only 4.9x (objActor) and 9.3x (criticLoss) more than the fp32 arm.  They are held to
    # the fp32 criterion alone; the tensors they are formed from and the gradients carry the TF32 one.
    for key in ("objActor", "criticLoss"):
        cmp(key, lrn.last[key], sharp=False)
    # The weight gradient of the 256 -> 7 layer contracts over the 20 480 rows of its input relu(h), which the 3xTF32
    # GEMM computes (check_gemm: the tensor core reads the lo terms truncated, an error of one sign per product).
    # Measured on an H100 SXM (700 W): 1.7e-5 of max|ref64|, 21x the fp32 arm's 8.2e-7 and 24x below TF32's 4.2e-4;
    # R2D2's second layers, over 3 840 rows, measure 6x and 13x.  The 2592 -> 256 GEMM itself stays within 0.12 of its
    # per-element bound on the same step (test_impala_step_kernels_on_their_inputs).
    cmp.grads(spies.grads, k={"module01.MLP_2.weight": 32})
    cmp.check()


def test_r2d2_step_against_fp64(R, L, monkeypatch):
    lrn, snap, spies, res = _r2d2_step(R, L, monkeypatch)
    _r2d2_compare(lrn, snap, spies, res)
    _close(lrn)


def test_impala_step_against_fp64(R, L, monkeypatch):
    lrn, snap, spies = _impala_step(R, L, monkeypatch)
    _impala_compare(lrn, snap, spies)
    _close(lrn)


def test_r2d2_comparison_sees_the_target_net_reading_online_weights(R, L, monkeypatch):
    """Negative control: the target pack's net 1 (the target net's conv_1) packed from the online weights."""
    def fault(mp, lrn):
        pack = R.Conv1Pack.pack
        w_on = getattr(lrn.model, lrn.model.first_conv_node()).conv_1.weight

        def online_for_target(p, net, weight):
            return pack(p, net, w_on if (p.n_nets == 2 and net == 1) else weight)
        mp.setattr(R.Conv1Pack, "pack", online_for_target)

    lrn, snap, spies, res = _r2d2_step(R, L, monkeypatch, fault)
    with pytest.raises(AssertionError, match="q_target"):
        _r2d2_compare(lrn, snap, spies, res)
    _close(lrn)


def test_impala_comparison_sees_the_bootstrap_one_step_early(R, L, monkeypatch):
    """Negative control: conv_1's bootstrap block (the last B rows) replaced by the B rows before it, time step
    T - 1."""
    def fault(mp, lrn):
        conv = R.conv1_fused
        TB, B = lrn.cfg.UNROLL_STEP * lrn.cfg.BATCHSIZE, lrn.cfg.BATCHSIZE

        def boot_one_step_early(*a, **k):
            out = conv(*a, **k)
            out[0][TB:].copy_(out[0][TB - B:TB])
            return out
        mp.setattr(R, "conv1_fused", boot_one_step_early)

    lrn, snap, spies = _impala_step(R, L, monkeypatch, fault)
    with pytest.raises(AssertionError, match="boot"):
        _impala_compare(lrn, snap, spies)
    _close(lrn)


# --------------------------------------------------------------------------- #
# C. the target kernels at their edges                                         #
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("T,B", [(1, 1), (20, 1024), (20, 129), (100, 7)])
def test_vtrace_edges_against_fp64(R, T, B):
    """pi from 1e-30 to 1, pi = mu, pi / mu far above and below the clips, zero bootstraps; every c_bar, p_bar in
    {0.5, 1, 2} and lambda in {0.95, 1}."""
    x = [torch.from_numpy(a).cuda() for a in vtrace_inputs(T, B, 100 * T + B)]
    for cbar in (0.5, 1.0, 2.0):
        for pbar in (0.5, 1.0, 2.0):
            for lam in (0.95, 1.0):
                vt, adv = R.vtrace(*x, 0.99, lam, cbar, pbar)
                check_vtrace(f"vtrace c={cbar} p={pbar} lambda={lam}", *x, 0.99, lam, cbar, pbar, vt, adv)


R2D2_EDGES = {
    "n=1": dict(L=60, B=64, n=1),
    "n=L-2": dict(L=10, B=5, n=8),
    "n=31": dict(L=60, B=8, n=31),
    "L=300": dict(L=300, B=3, n=5),
    "B=1": dict(L=60, B=1, n=5),
    "Q=1e4": dict(L=60, B=16, n=5, scale=1e4),
    "Q=0": dict(L=60, B=16, n=5, scale=0.0),
    "Q subnormal": dict(L=60, B=16, n=5, scale=1e-40),
    "notdone=0, zero weights": dict(L=60, B=16, n=5, terminal=True),
}


@pytest.mark.parametrize("rescale", [True, False])
@pytest.mark.parametrize("case", list(R2D2_EDGES))
def test_r2d2_target_edges_bit_for_bit(R, case, rescale):
    """b2rl_r2d2_target against oracle.r2d2_target: target, td and grad_q bit for bit, prio and the scalars at
    test_gpu_00's tolerances."""
    e = R2D2_EDGES[case]
    L_, B, A, n = e["L"], e["B"], 6, e["n"]
    rng = np.random.default_rng(L_ * 1000 + B + n)
    scale = e.get("scale", 3.0)
    q = (rng.standard_normal((L_, B, A)) * scale).astype(np.float32)
    qt = (rng.standard_normal((L_, B, A)) * scale).astype(np.float32)
    a = rng.integers(0, A, size=(L_ - 1, B))
    r = rng.standard_normal((L_ - 1, B)).astype(np.float32)
    nd = np.zeros(B, np.float32) if e.get("terminal") else (rng.random(B) > 0.3).astype(np.float32)
    w = rng.uniform(0.1, 1, size=B).astype(np.float32)
    if e.get("terminal"):
        w[::2] = 0.0
    dev = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (q, qt, a, r, nd, w)]
    out = R.r2d2_target(*dev, n, 0.997, 0.9, rescale)
    tgt, td, prio, gq, info = O.r2d2_target(q, qt, a, r, nd, w, n, 0.997, 0.9, rescale)
    for name, ref in (("target", tgt), ("td", td), ("grad_q", gq)):
        got = out[name].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (case, name)
    np.testing.assert_allclose(out["prio"].cpu().numpy(), prio, rtol=5e-7)
    np.testing.assert_allclose(out["scalars"].cpu().numpy(), [info["loss"], info["mean_value"]], rtol=2e-6, atol=1e-7)


def test_r2d2_target_refuses_n_32(R):
    """n = 32 is beyond the kernel's table of gamma powers (R2D2_MAX_NSTEP): refused with B2RL_ERR_INVALID, nothing
    launched."""
    from distributed_rl_b200 import _lib
    lib = _lib.load()
    L_, B, A = 60, 4, 6
    q = torch.zeros(L_, B, A, device="cuda")
    a = torch.zeros(L_ - 1, B, dtype=torch.int64, device="cuda")
    r = torch.zeros(L_ - 1, B, device="cuda")
    v = torch.ones(B, device="cuda")
    outs = [torch.empty(L_ - 1, B, device="cuda"), torch.empty(L_ - 1, B, device="cuda"), torch.empty(B, device="cuda"),
            torch.empty(L_, B, A, device="cuda"), torch.empty(2, device="cuda")]
    n0 = lib.b2rl_launch_count()
    for n_step, ok in ((31, True), (32, False)):
        rc = lib.b2rl_r2d2_target(q.data_ptr(), q.data_ptr(), a.data_ptr(), r.data_ptr(), v.data_ptr(), v.data_ptr(),
                                  L_, B, A, n_step, 0.997, 0.9, 1, *(t.data_ptr() for t in outs),
                                  torch.cuda.current_stream().cuda_stream)
        assert (rc == 0) == ok, (n_step, rc)
    torch.cuda.synchronize()
    assert lib.b2rl_launch_count() == n0 + 2, "n = 31 is two launches (target + scalars), n = 32 none"
