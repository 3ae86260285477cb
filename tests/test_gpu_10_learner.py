"""GPU tests of the reference-facing Ape-X mirror (distributed_rl_b200/apex.py):
Learner.train against the reference's loss/backward math written with plain
autograd, and the CUDA-graph fused step against the eager step."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def apex():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cudnn.allow_tf32 = False      # fp32 everywhere so both paths round alike
    torch.backends.cuda.matmul.allow_tf32 = False
    from distributed_rl_b200 import apex
    return apex


def _mk(apex, B=32, N=4096, seed=0, **kw):
    cfg = apex.ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                          CUDNN_BENCHMARK=False, **kw)
    torch.manual_seed(seed)
    L = apex.Learner(cfg, connect=None, start_replay=False)
    with torch.no_grad():
        for p in L.target_model.parameters():
            p.add_(0.01 * torch.randn(p.shape, device=p.device))    # by logical index: independent of the memory format
    return cfg, L


def _fill(L, N, seed=1):
    st = L.memory.store
    st.fill_hash(N, seed=seed)
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    st.field_view("action").copy_(torch.randint(0, 6, (N,), device="cuda", generator=g, dtype=torch.int32))
    st.field_view("reward").copy_(torch.randn(N, device="cuda", generator=g).clamp_(-1, 1))
    st.field_view("done").copy_((torch.rand(N, device="cuda", generator=g) < 0.1).to(torch.uint8))
    st.build((torch.randn(N, device="cuda", generator=g).abs().clamp(max=1) + 1e-7) ** 0.6)
    st.seed(99, 0)


def test_train_matches_reference_math_with_autograd(apex):
    """Learner.train (fused target kernel + dLoss/dQ seeding) == APE_X/Learner.py:55-121 written
    with torch ops and loss.backward(), on the same weights and minibatch."""
    cfg, L = _mk(apex, B=32)
    _fill(L, 4096)
    batch = L.memory.sample()
    s, a, r, ns, d, w, idx = batch
    # reference math on a deep copy of the networks
    import copy
    ref_model, ref_target = copy.deepcopy(L.model), copy.deepcopy(L.target_model)
    ref_opt = apex.make_optimizer(cfg.OPTIM_INFO, ref_model.getParameters(), capturable=False)
    sf, nsf = s.float() / 255., ns.float() / 255.
    q = ref_model.forward([sf])[0]
    with torch.no_grad():
        qt = ref_target.forward([nsf])[0]
        qn = ref_model.forward([nsf])[0]
        a_star = qn.argmax(-1)
        nxt = qt.gather(1, a_star[:, None])[:, 0] * (1 - d.float())
    q_sa = q.gather(1, a.long()[:, None])[:, 0]
    target = r + 0.99 ** cfg.UNROLL_STEP * nxt
    td = torch.clamp(target - q_sa, -1, 1)
    prio_ref = (td.detach().abs().cpu().numpy() + 1e-7) ** cfg.ALPHA
    loss = torch.mean(w * td ** 2) * 0.5
    loss.backward()
    gref = [p.grad.clone() for p in ref_model.parameters()]
    ref_opt.step()

    info, prio, idx2, mean_w = L.train(batch)
    for p, pr, g in zip(L.model.parameters(), ref_model.parameters(), gref):
        np.testing.assert_allclose(p.detach().cpu().numpy(), pr.detach().cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(prio.cpu().numpy(), prio_ref, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(float(info["loss"]), float(loss.detach()), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(float(info["mean_value"]), float(target.mean()), atol=1e-5)
    np.testing.assert_allclose(float(mean_w), float(w.mean()), atol=1e-6)
    assert torch.equal(idx2, idx)


def test_train_accepts_reference_host_transition(apex):
    """The reference passes numpy object arrays (APE_X/ReplayMemory.py:87-113); same call works."""
    cfg, L = _mk(apex, B=8)
    rng = np.random.default_rng(0)
    s = rng.integers(0, 256, size=(8, 4, 84, 84), dtype=np.uint8)
    ns = rng.integers(0, 256, size=(8, 4, 84, 84), dtype=np.uint8)
    a = np.array([int(x) for x in rng.integers(0, 6, size=8)], dtype=object)
    r = np.array([float(x) for x in rng.standard_normal(8)], dtype=object)
    d = np.array([bool(x) for x in rng.random(8) < 0.3], dtype=object)
    w = torch.rand(8); idx = torch.arange(8)
    info, prio, idx2, mw = L.train([s, a, r, ns, d, w, idx])
    assert prio.shape == (8,) and torch.isfinite(prio).all()
    L.memory.store.build(torch.ones(64, device="cuda"))
    L.memory.update(list(idx2), prio.cpu().numpy())     # reference call: list of 0-d tensors + ndarray
    np.testing.assert_allclose(L.memory.store.priorities(0, 8).cpu().numpy(), prio.cpu().numpy())


def _rel(a, b):
    """norm-wise relative difference ||a - b|| / ||b|| (fp64 accumulate)."""
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def test_fused_graph_step_equals_eager_step(apex):
    """5 fused steps as a CUDA graph == 5 eager fused steps (same seeds, same kernels, cuDNN heuristics +
    deterministic algorithms): the same slots are sampled and the weights moved by the same update.
    Compared norm-wise against the size of the UPDATE (centred RMSprop's early step is ~lr*sign(g)/0.22,
    so an element-wise comparison of weights is ill-conditioned wherever g ~ 0)."""
    res = []
    for use_graph in (False, True):
        cfg, L = _mk(apex, B=64, N=8192, seed=3)
        init = [p.detach().clone() for p in L.model.parameters()]
        _fill(L, 8192, seed=5)
        for _ in range(5 if not use_graph else 1):
            out = L.fused_step(use_graph=use_graph)
        if use_graph:   # building the graph ran 3 warm-ups + capture(=no execution) + 1 replay = 4 bodies
            L.fused_step(use_graph=True)
        torch.cuda.synchronize()
        res.append(([p.detach().clone() for p in L.model.parameters()], L.memory.store.priorities().clone(),
                    L.launches_per_step, init, out["idx"].clone()))
    (pe, te, le, init, ie), (pg, tg, lg, _, ig) = res
    assert torch.equal(ie, ig)                    # step 5 sampled the same slots from the same tree
    for a, b, w0 in zip(pe, pg, init):
        assert _rel(a - w0, b - w0) <= 1e-3       # same update (bit-equal kernels; bound leaves room for cuDNN)
    assert (te != tg).float().mean() < 0.01       # same slots updated with (nearly) the same priorities
    assert le == lg and le >= 4                   # sample, gather, target, update (+conv1/optimizer kernels)


def test_r2d2_learner_train_matches_oracle_and_autograd():
    """R2D2 mirror: priorities == oracle on the captured Q tensors; the parameter update equals
    loss.backward() of 0.5*mean(w*(y - q_sa)^2) (R2D2/Learner.py:184-192) + clip 40 + Adam."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import copy
    from oracle import oracle as O
    from distributed_rl_b200 import r2d2
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    T, MEM, B = 16, 8, 4
    cfg = r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=MEM, REPLAY_MEMORY_LEN=64, BUFFER_SIZE=0)
    torch.manual_seed(0)
    L = r2d2.Learner(cfg)
    with torch.no_grad():
        for p in L.target_model.parameters():
            p.add_(0.02 * torch.randn(p.shape, device=p.device))
    ref_model = copy.deepcopy(L.model)
    ref_opt = r2d2.make_optimizer(cfg.OPTIM_INFO, ref_model.getParameters(), capturable=False)
    rng = np.random.default_rng(0)
    n = 64
    L.memory.push_arrays(rng.integers(0, 256, size=(n, T, 4, 84, 84), dtype=np.uint8),
                         rng.integers(0, 6, size=(n, T)).astype(np.int32),
                         rng.standard_normal((n, T)).astype(np.float32),
                         (rng.standard_normal((n, 512)) * 0.1).astype(np.float32),
                         (rng.standard_normal((n, 512)) * 0.1).astype(np.float32),
                         (rng.random(n) > 0.3).astype(np.float32), rng.uniform(0.1, 1, n).astype(np.float32))
    batch = L.memory.sample()
    (h0, h1), s, a, r, nd, w, idx = batch
    cap = {}
    om, ot = L.model.forward, L.target_model.forward

    def fm(x, **kw):
        o = om(x, **kw); cap.setdefault("q", []).append(o[0]); return o

    def ft(x, **kw):
        o = ot(x, **kw); cap.setdefault("qt", []).append(o[0]); return o

    L.model.forward, L.target_model.forward = fm, ft
    info, prio, idx2 = L.train(batch)
    Lw = T - MEM
    q = cap["q"][1].detach().view(Lw, B, 6).cpu().numpy()
    qt = cap["qt"][1].detach().view(Lw, B, 6).cpu().numpy()
    act = a.t()[MEM:-1].cpu().numpy(); rew = r.t()[MEM:-1].cpu().numpy()
    tgt, td, oprio, gq, oinfo = O.r2d2_target(q, qt, act, rew, nd.cpu().numpy(), w.cpu().numpy(),
                                              cfg.UNROLL_STEP, cfg.GAMMA, cfg.ALPHA, True)
    np.testing.assert_allclose(prio.cpu().numpy(), oprio, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(float(info["mean_value"]), oinfo["mean_value"], atol=1e-6)
    # autograd restatement on the copy
    ref_model.setCellState((h0, h1))
    sf = (s.float() / 255.).permute(1, 0, 2, 3, 4).contiguous()
    with torch.no_grad():
        ref_model.forward([sf[:MEM].reshape(-1, 4, 84, 84), torch.tensor([MEM, B, -1])])
        ref_model.detachCellState()
    qr = ref_model.forward([sf[MEM:].reshape(-1, 4, 84, 84), torch.tensor([Lw, B, -1])])[0].view(Lw, B, 6)
    sel = qr[:-1].gather(2, a.t()[MEM:-1].long().unsqueeze(-1))[..., 0]
    loss = torch.mean(w.view(1, -1) * (torch.from_numpy(tgt).cuda() - sel) ** 2) * 0.5
    loss.backward()
    torch.nn.utils.clip_grad_norm_(ref_model.getParameters(), 40)
    ref_opt.step()
    for p, pr in zip(L.model.parameters(), ref_model.parameters()):
        np.testing.assert_allclose(p.detach().cpu().numpy(), pr.detach().cpu().numpy(), rtol=1e-4, atol=2e-6)
    L.memory.update(list(idx2), prio)
    np.testing.assert_allclose(L.memory.store.priorities()[idx2].cpu().numpy(), prio.cpu().numpy())


def test_impala_learner_train_matches_oracle():
    """IMPALA mirror: V-trace targets/advantages == oracle on the learner's own pi, V; params move."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import oracle as O
    from distributed_rl_b200 import impala
    torch.backends.cudnn.allow_tf32 = False
    T, B, n = 20, 8, 32
    cfg = impala.ImpalaConfig(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=n, BUFFER_SIZE=0)
    torch.manual_seed(1)
    L = impala.Learner(cfg)
    rng = np.random.default_rng(1)
    L._memory.push_arrays(rng.integers(0, 256, size=(n, T + 1, 28224), dtype=np.uint8),
                          rng.integers(0, 6, size=(n, T)).astype(np.int32),
                          rng.uniform(0.05, 0.9, size=(n, T)).astype(np.float32),
                          rng.standard_normal((n, T)).astype(np.float32),
                          (rng.random(n) > 0.3).astype(np.float32))
    tr = L._memory.sample()
    s, a, mu, r, done = tr
    assert s.shape == (T + 1, B, 28224) and a.shape == (T, B)
    with torch.no_grad():
        sf = (s.float() / 255.).view(T + 1, B, 4, 84, 84)
        boot = L.model.forward([sf[-1]])[0][:, -1] * done
        pi_a, v = L.forward(sf[:-1].reshape(-1, 4, 84, 84), a.reshape(-1))
    before = [p.detach().clone() for p in L.model.parameters()]
    L.train(tr, 0)
    ovt, oadv, _ = O.vtrace(pi_a.view(T, B).cpu().numpy(), mu.cpu().numpy(), v.view(T, B).cpu().numpy(),
                            boot.cpu().numpy(), r.cpu().numpy(), cfg.GAMMA, cfg.C_LAMBDA, cfg.C_VALUE, cfg.P_VALUE)
    np.testing.assert_allclose(L.last["vtarget"].cpu().numpy(), ovt, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(L.last["advantage"].cpu().numpy(), oadv, rtol=1e-5, atol=1e-5)
    assert any((b != p).any().item() for b, p in zip(before, L.model.parameters()))
    assert all(torch.isfinite(p).all().item() for p in L.model.parameters())


def _first_step_gradients(apex, fused, B=64, N=8192, **kw):
    """Gradients (before the optimizer) of one Ape-X step on the slots the device RNG draws."""
    cfg, L = _mk(apex, B=B, N=N, seed=11, FUSED_CONV1=fused, **kw)
    _fill(L, N, seed=5)
    st = L.memory.store
    idx, _, w = st.sample(B, beta=cfg.BETA, want_prob=False)
    if fused:
        assert L._conv1_ready()
        b = st.gather(idx, st.alloc_batch(B, ("action", "reward", "done")))
        out = L._forward_backward_fused(idx, b["action"].to(torch.int64), b["reward"], b["done"], w)
    else:
        b = st.gather(idx)
        out = L._forward_backward(b["state"], b["action"].to(torch.int64), b["reward"], b["next_state"], b["done"], w)
    torch.cuda.synchronize()
    return L, idx.clone(), out, [p.grad.detach().clone() for p in L.model.parameters()]


def test_fused_conv1_gradients_equal_staged_gradients(apex):
    """The benchmarked path (wgmma gather+conv_1 forward and weight gradient, 3xTF32 heads, fused dueling tail,
    weight gradients on the side stream) against the staged path (gathered uint8 batch -> fp32 -> cuDNN fp32 conv_1):
    same sampled slots, TD errors / priorities to fp32 noise, and every parameter's GRADIENT equal norm-wise
    (||dg|| / ||g|| <= 2e-5).  Gradients, not post-RMSprop weights: the centred RMSprop step is ~lr*sign(g)/0.22
    wherever g ~ 0, which turns 1e-6 input noise into sign flips (the round-1 flake)."""
    L0, i0, o0, g0 = _first_step_gradients(apex, False)
    L1, i1, o1, g1 = _first_step_gradients(apex, True)
    assert torch.equal(i0, i1)                                   # same device RNG stream, same tree
    np.testing.assert_allclose(o1["td"].cpu().numpy(), o0["td"].cpu().numpy(), rtol=0, atol=1e-5)
    np.testing.assert_allclose(o1["prio"].cpu().numpy(), o0["prio"].cpu().numpy(), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(o1["scalars"].cpu().numpy(), o0["scalars"].cpu().numpy(), rtol=1e-5, atol=1e-6)
    names = [n for n, _ in L0.model.named_parameters()]
    for n, a, b in zip(names, g1, g0):
        assert b.abs().max() > 0, n
        r = _rel(a, b)
        assert r <= 2e-5, (n, r)


def test_batched_online_pass_equals_separate_passes(apex):
    """BATCHED_ONLINE: Q(s) and Q_online(s') as ONE B = 2*BATCHSIZE pass recorded on an OutputTape, the autograd graph
    of the s half built by replaying the recorded outputs — against the three separate passes: same TD errors and
    priorities, every gradient equal norm-wise (cuDNN may pick another algorithm at the doubled batch: 2e-5)."""
    L0, i0, o0, g0 = _first_step_gradients(apex, True, BATCHED_ONLINE=False)
    L1, i1, o1, g1 = _first_step_gradients(apex, True, BATCHED_ONLINE=True)
    assert torch.equal(i0, i1)
    np.testing.assert_allclose(o1["td"].cpu().numpy(), o0["td"].cpu().numpy(), rtol=0, atol=1e-5)
    np.testing.assert_allclose(o1["prio"].cpu().numpy(), o0["prio"].cpu().numpy(), rtol=1e-4, atol=1e-6)
    for n, a, b in zip([n for n, _ in L0.model.named_parameters()], g1, g0):
        r = _rel(a, b)
        assert r <= 2e-5, (n, r)


def test_fused_conv1_steps_move_weights_like_staged_steps(apex):
    """Three whole fused_step()s (sample -> ... -> RMSprop -> priority write-back) on both paths: the same slots
    are drawn at step 3 (the trees evolved alike) and the accumulated weight UPDATE agrees norm-wise to 5 % (sign
    flips of near-zero gradients under centred RMSprop are allowed, a wrong kernel is not)."""
    res = []
    for fused in (False, True):
        cfg, L = _mk(apex, B=64, N=8192, seed=11, FUSED_CONV1=fused)
        init = [p.detach().clone() for p in L.model.parameters()]
        _fill(L, 8192, seed=5)
        outs = [L.fused_step(use_graph=False) for _ in range(3)]
        torch.cuda.synchronize()
        res.append(([p.detach().clone() for p in L.model.parameters()], L.memory.store.priorities().clone(),
                    outs[-1]["idx"].clone(), outs[-1]["scalars"].clone(), init))
    (p0, t0, i0, s0, init), (p1, t1, i1, s1, _) = res
    assert torch.equal(i0, i1)
    np.testing.assert_allclose(s0.cpu().numpy(), s1.cpu().numpy(), rtol=1e-3, atol=1e-5)
    assert ((t0 - t1).abs() > 1e-3 * t0.abs() + 1e-5).float().mean() < 0.01
    for a, b, w0 in zip(p1, p0, init):
        assert _rel(a - w0, b - w0) <= 5e-2


@pytest.mark.parametrize("centered,eps,alpha", [(True, 1.5e-7, 0.95), (False, 1e-5, 0.99)])
def test_fused_rmsprop_matches_torch_optim(centered, eps, alpha):
    """csrc/optim.cu == torch.optim.RMSprop (the optimiser getOptim builds, baseline/utils.py:124-130)
    over 4 steps, including a channels_last conv weight; plus zero_grad and the reference's 'norm'."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200.optim import FusedRMSprop
    torch.manual_seed(0)
    shapes = [(32, 4, 8, 8), (64, 32, 4, 4), (512, 3136), (6, 512), (1, 7)]
    mine = [torch.randn(s, device="cuda") * 0.1 for s in shapes]
    mine[1] = mine[1].contiguous(memory_format=torch.channels_last)
    ref = [p.detach().clone(memory_format=torch.preserve_format).requires_grad_(True) for p in mine]
    mine = [p.requires_grad_(True) for p in mine]
    opt_ref = torch.optim.RMSprop(ref, lr=6.25e-5, alpha=alpha, eps=eps, centered=centered)
    opt = FusedRMSprop(mine, lr=6.25e-5, alpha=alpha, eps=eps, centered=centered)
    for step in range(4):
        gs = [torch.randn_like(p) * (0.5 + step) for p in ref]
        for p, q, g in zip(ref, mine, gs):
            p.grad = g.clone(memory_format=torch.preserve_format)
            q.grad.copy_(g)
        want_norm = sum(g.norm(2) for g in gs) ** 0.5
        norm = opt.step()
        opt_ref.step()
        np.testing.assert_allclose(float(norm), float(want_norm), rtol=1e-6)
        for p, q in zip(ref, mine):
            np.testing.assert_allclose(q.detach().cpu().numpy(), p.detach().cpu().numpy(), rtol=2e-6, atol=2e-8)
            assert float(q.grad.abs().max()) == 0.0            # zero_grad fused


def test_fused_rmsprop_early_late_split_equals_one_step():
    """The optimizer step issued in two parts (dense heads early, the rest + the 'norm' later: optim.set_early /
    step_early / step, b2rl_rmsprop_norm_finish) is bit-identical to the single launch — parameters, optimizer state,
    zeroed gradients — and gives the same 'norm' (APE_X/Learner.py:123-138 has no cross-parameter term)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200.optim import FusedRMSprop
    torch.manual_seed(1)
    shapes = [(32, 4, 8, 8), (64, 32, 4, 4), (512, 3136), (6, 512), (512, 3136), (1, 512)]
    a = [(torch.randn(s, device="cuda") * 0.1).requires_grad_(True) for s in shapes]
    b = [p.detach().clone().requires_grad_(True) for p in a]
    one = FusedRMSprop(a, lr=6.25e-5, alpha=0.95, eps=1.5e-7, centered=True)
    two = FusedRMSprop(b, lr=6.25e-5, alpha=0.95, eps=1.5e-7, centered=True)
    assert not two.set_early([b[0], b[2]])            # not a contiguous run: refused, nothing changes
    assert two.set_early(b[2:])
    side = torch.cuda.Stream()
    for step in range(3):
        gs = [torch.randn(s, device="cuda") * (0.5 + step) for s in shapes]
        for p, q, g in zip(a, b, gs):
            p.grad.copy_(g)
            q.grad.copy_(g)
        n1 = one.step().clone()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            two.step_early()
        torch.cuda.current_stream().wait_stream(side)
        n2 = two.step().clone()
        np.testing.assert_allclose(float(n2), float(n1), rtol=1e-6)      # fp64 atomics: order-dependent at 1e-16
        assert float(n1) > 0
        for p, q, s1, s2, g1, g2 in zip(a, b, one.square_avg, two.square_avg, one.grad_avg, two.grad_avg):
            assert torch.equal(p, q) and torch.equal(s1, s2) and torch.equal(g1, g2)
            assert float(q.grad.abs().max()) == 0.0


@pytest.mark.parametrize("fused", [False, True])
def test_learner_train_end_to_end_vs_reference_golden(apex, golden, fused):
    """The whole reference Learner.train (run on the CPU by tests/golden/make_golden.py: 3 forwards,
    double-DQN target, clipped TD, priority, IS-weighted loss, backward, centered RMSprop) against
    distributed_rl_b200.apex.Learner.train on the GPU with the same seeded weights and minibatch.
    `fused` routes conv_1 through the wgmma kernel via an in-replay batch and fused_step."""
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_golden import seeded_weights
    g = golden("apex_e2e")
    B = int(g["batch"])
    cfg = apex.ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=64, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                          FUSED_CONV1=fused, CUDNN_BENCHMARK=False)
    L = apex.Learner(cfg, connect=None, start_replay=False)
    for model, seed, tag in ((L.model, 101, "online"), (L.target_model, 202, "target")):
        names = [str(n) for n in g[f"{tag}_names"]]
        sd = model.state_dict()
        assert list(sd.keys()) == names                       # same state_dict key order as the reference
        ws = seeded_weights([tuple(sd[k].shape) for k in names], seed)
        model.load_state_dict({k: torch.from_numpy(w) for k, w in zip(names, ws)})
    rng = np.random.default_rng(0xB200 + 99)                   # same draws as gen_apex_e2e
    s = rng.integers(0, 256, size=(B, 4, 84, 84), dtype=np.uint8)
    ns = rng.integers(0, 256, size=(B, 4, 84, 84), dtype=np.uint8)
    a = np.array([int(x) for x in rng.integers(0, 6, size=B)], dtype=object)
    r = np.array([float(x) for x in np.clip(rng.standard_normal(B), -1, 1)], dtype=object)
    d = np.array([bool(x) for x in (rng.random(B) < 0.25)], dtype=object)
    w = torch.from_numpy(rng.uniform(0.2, 1.0, size=B).astype(np.float32))
    if not fused:
        info, prio, idx, mean_w = L.train([s, a, r, ns, d, w, torch.arange(B)])
        prio = prio.cpu().numpy(); mean_value = float(info["mean_value"]); p_norm = float(info["p_norm"])
    else:
        # put exactly this minibatch into the replay, sample it with explicit uniforms in order
        st = L.memory.store
        st.push([s, ns, a.astype(np.int32), r.astype(np.float32), d.astype(np.uint8)], np.ones(B, np.float32))
        idx = torch.arange(B, device="cuda")
        L._conv1_ready()
        out = L._forward_backward_fused(idx, torch.from_numpy(a.astype(np.int64)).cuda(),
                                        torch.from_numpy(r.astype(np.float32)).cuda(),
                                        torch.from_numpy(d.astype(np.uint8)).cuda(), w.cuda())
        info = L.step()
        prio = out["prio"].cpu().numpy(); mean_value = float(out["scalars"][1]); p_norm = float(info["p_norm"])
    np.testing.assert_allclose(prio, g["new_priority"], rtol=2e-4, atol=2e-5)     # Q-values through a CPU vs GPU net
    np.testing.assert_allclose(mean_value, float(g["mean_value"]), atol=2e-5)
    np.testing.assert_allclose(p_norm, float(g["p_norm"]), rtol=1e-3)
    for k, v in L.model.state_dict().items():
        got = v.reshape(-1)[:256].cpu().numpy() if v.is_contiguous() else v.contiguous().reshape(-1)[:256].cpu().numpy()
        # centered RMSprop's first step is ~ lr*sign(g)/0.218: insensitive to |g|, so 1e-6 absolute
        np.testing.assert_allclose(got, g["after_" + k], rtol=0, atol=2e-6, err_msg=k)


def _golden_tools():
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden
    return make_golden


def test_r2d2_learner_train_end_to_end_vs_reference_golden(golden):
    """Reference R2D2 Learner.train on the CPU (burn-in, LSTM, n-step targets with h / h^-1, clip 40,
    Adam) vs distributed_rl_b200.r2d2.Learner.train on the GPU, seeded weights + sequences."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import r2d2
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    mg = _golden_tools()
    g = golden("r2d2_e2e")
    T, MEM, B = [int(x) for x in g["dims"]]
    cfg = r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=MEM, REPLAY_MEMORY_LEN=16, BUFFER_SIZE=0)
    L = r2d2.Learner(cfg)
    assert mg._load_seeded(L.model, 303) == [str(n) for n in g["online_names"]]
    assert mg._load_seeded(L.target_model, 404) == [str(n) for n in g["target_names"]]
    L.model.cuda(); L.target_model.cuda()
    rng = np.random.default_rng(0xB200 + 77)
    s = rng.integers(0, 256, size=(B, T, 4, 84, 84), dtype=np.uint8)
    a = rng.integers(0, 6, size=(B, T)).astype(np.int32)
    r = rng.standard_normal((B, T)).astype(np.float32)
    notdone = np.array([float(x) for x in (rng.random(B) > 0.3)])
    w = torch.from_numpy(rng.uniform(0.2, 1.0, size=B).astype(np.float32))
    h0 = torch.from_numpy((rng.standard_normal((1, B, 512)) * 0.1).astype(np.float32))
    h1 = torch.from_numpy((rng.standard_normal((1, B, 512)) * 0.1).astype(np.float32))
    info, prio, idx = L.train([(h0, h1), torch.from_numpy(s), torch.from_numpy(a), torch.from_numpy(r),
                               torch.from_numpy(notdone.astype(np.float32)), w, torch.arange(B)])
    np.testing.assert_allclose(prio.cpu().numpy(), g["new_priority"], rtol=5e-4, atol=5e-5)
    np.testing.assert_allclose(float(info["mean_value"]), float(g["mean_value"]), atol=5e-5)
    np.testing.assert_allclose(float(info["p_norm"]), float(g["p_norm"]), rtol=2e-3)
    for k, v in L.model.state_dict().items():
        np.testing.assert_allclose(v.contiguous().reshape(-1)[:256].cpu().numpy(), g["after_" + k], rtol=0, atol=5e-6,
                                   err_msg=k)


def test_impala_learner_train_end_to_end_vs_reference_golden(golden):
    """Reference IMPALA Learner.train on the CPU (V-trace, actor/critic/entropy loss, clip 40, RMSprop)
    vs distributed_rl_b200.impala.Learner.train on the GPU."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import impala
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    mg = _golden_tools()
    g = golden("impala_e2e")
    T, B = [int(x) for x in g["dims"]]
    cfg = impala.ImpalaConfig(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=16, BUFFER_SIZE=0)
    L = impala.Learner(cfg)
    assert mg._load_seeded(L.model, 505) == [str(n) for n in g["names"]]
    L.model.cuda()
    rng = np.random.default_rng(0xB200 + 55)
    s = rng.integers(0, 256, size=(T + 1, B, 4 * 84 * 84), dtype=np.uint8)
    a = rng.integers(0, 6, size=(T, B)).astype(np.int64)
    mu = rng.uniform(0.05, 0.9, size=(T, B)).astype(np.float32)
    r = rng.standard_normal((T, B)).astype(np.float32)
    done = (rng.random(B) > 0.3).astype(np.float32)
    L.train((s, a, mu, r, done), 0)
    for k, v in L.model.state_dict().items():
        # RMSprop (lr 6e-4, eps 1e-5): first step ~ lr * g / (0.1|g| + eps), so compare to 1e-5 absolute
        np.testing.assert_allclose(v.contiguous().reshape(-1)[:256].cpu().numpy(), g["after_" + k], rtol=0, atol=1e-5,
                                   err_msg=k)


def test_async_parameter_publication_and_run_loop(apex):
    """Learner.run publishes `state_dict` / `count` / `target_state_dict` under the reference's Redis
    keys (APE_X/Learner.py:149-155,207-216) through the async publisher; payload = dict of CPU tensors
    with the reference's key names, equal to the weights at the snapshot step."""
    import pickle
    from oracle.ref_harness import _StrictRedis
    from distributed_rl_b200.publish import ParamPublisher
    cfg = apex.ApexConfig(BATCHSIZE=32, REPLAY_MEMORY_LEN=4096, BUFFER_SIZE=0, TARGET_FREQUENCY=60,
                          LEARNER_DEVICE="cuda:0", CUDNN_BENCHMARK=False)
    conn = _StrictRedis()
    L = apex.Learner(cfg, connect=conn, start_replay=False)
    _fill(L, 4096)
    # publisher alone: snapshot -> poll(block) reproduces the weights bit-exactly
    pub = ParamPublisher(L.model, conn, "state_dict", "count")
    pub.snapshot(7)
    assert pub.poll(block=True)
    sd = pickle.loads(conn.get("state_dict"))
    assert pickle.loads(conn.get("count")) == 7
    for k, v in L.model.state_dict().items():
        assert torch.equal(sd[k], v.cpu())
    steps = L.run(max_steps=120, log_every=10 ** 9)
    assert steps == 120
    for p in L._publishers:
        p.poll(block=True)
    assert L._publishers[0].published >= 1 and L._publishers[1].published >= 1
    assert set(pickle.loads(conn.get("target_state_dict"))) == set(L.model.state_dict())
    assert pickle.loads(conn.get("count")) in (0, 50)


def test_push_records_decodes_actor_blobs_through_pinned_staging(apex):
    """Replay.push_records: pickled [s, a, R_n, s', done, prio] records (APE_X/Player.py:252-261) land in the
    ring in order, through the NUMA-local pinned staging sets (two alternating sets, grown on demand)."""
    import pickle
    from distributed_rl_b200 import hostmem
    cfg, L = _mk(apex, B=32, N=1024, seed=1)
    rng = np.random.default_rng(0)
    mem = L.memory
    recs_all = []
    for n in (5, 70, 3):                         # second call grows the staging set, third reuses the first
        recs = [[rng.integers(0, 256, size=(4, 84, 84), dtype=np.uint8), int(rng.integers(0, 6)),
                 float(rng.standard_normal()), rng.integers(0, 256, size=(4, 84, 84), dtype=np.uint8),
                 bool(rng.random() < 0.3), float(rng.random() + 0.1)] for _ in range(n)]
        mem.push_records([pickle.dumps(r) for r in recs])
        recs_all += recs
    torch.cuda.synchronize()
    st = mem.store
    assert len(st) == 78 and mem.total_frame == 78
    k = len(recs_all)
    np.testing.assert_array_equal(st.field_view("state")[:k].cpu().numpy().reshape(k, 4, 84, 84),
                                  np.stack([r[0] for r in recs_all]))
    np.testing.assert_array_equal(st.field_view("next_state")[:k].cpu().numpy().reshape(k, 4, 84, 84),
                                  np.stack([r[3] for r in recs_all]))
    np.testing.assert_array_equal(st.field_view("action")[:k].cpu().numpy().ravel(), [r[1] for r in recs_all])
    np.testing.assert_array_equal(st.field_view("reward")[:k].cpu().numpy().ravel(),
                                  np.asarray([r[2] for r in recs_all], np.float32))
    np.testing.assert_array_equal(st.field_view("done")[:k].cpu().numpy().ravel().astype(bool), [r[4] for r in recs_all])
    np.testing.assert_allclose(st.priorities()[:k].cpu().numpy(),
                               np.asarray([r[5] for r in recs_all], np.float32), rtol=0)   # stored as given (baseline/PER.py:69-75)
    # the staging pages are pinned; the NUMA binding is best-effort and must restore the thread's affinity
    import os
    before = os.sched_getaffinity(0)
    t = hostmem.pinned_empty((16,), torch.float32, "cuda:0")
    assert t.is_pinned() and os.sched_getaffinity(0) == before
