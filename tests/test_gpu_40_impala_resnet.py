"""GPU tests of the IMPALA residual network's fused stem (csrc/stem.cu: R.stem_fused, R.stem_wgrad) and of the IMPALA
learner on impala.resnet_small_model().

The stem forward against the restatement of its arithmetic (tests/stem_model.py) bit for bit, pooled values and
argmax, on random, constant and flat-block stacks (exact ties), borders included, at one stack per CTA and at three
or four per CTA through a permuting, repeating idx; against fp64 within check_stem's per-element bounds (each pooled
value within its own position's bound, each argmax within that bound of its window's maximum).  The weight gradient
within one fp32 ulp of the restatement and within check_stem_wgrad's per-element bound.  Both bit-identical across
runs and across frame sources holding the same frames.  The learner: fused_step against train() on the PyTorch stem;
the captured step against the eager one; the served captured step against the in-process one; dedup and coded stores
against a stack store."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stem_model as M                                          # noqa: E402
from fp64_bounds import check_stem, check_stem_wgrad            # noqa: E402
from impala_atari_rollouts import atari_rollouts                # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import replay
    return replay


@pytest.fixture(autouse=True)
def _deterministic():
    b = torch.backends
    saved = (b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32)
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = True, False, False, False
    yield
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = saved


def _stacks(n, seed):
    """n frame stacks (n >= 8): random, all-constant (0, 255, 77), flat blocks, and Atari-like frames."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, size=(n, 4, 84, 84), dtype=np.uint8)
    f[1], f[2], f[3] = 0, 255, 77
    blocks = rng.integers(0, 256, size=(4, 29, 29), dtype=np.uint8)
    f[4] = np.repeat(np.repeat(blocks, 3, axis=1), 3, axis=2)[:, :84, :84]
    state = atari_rollouts(4, T=2, actors=2, episode=(4, 12), p_done=0.1, seed=seed)[0]
    atari = state.reshape(-1, 4, 84, 84)
    f[5:] = atari[np.arange(n - 5) % len(atari)]
    return f


def _weights(seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(16, 4, 3, 3, generator=g) * scale


@pytest.fixture(scope="module")
def sms(R):
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_stem_forward_equals_the_model_bit_for_bit_and_fp64(R, sms):
    """n = 40: one stack per CTA.  Every stack bit for bit against stem_model's device restatement and its numpy loops,
    the constant stacks' tie rule, and against fp64 through check_stem's per-element bounds."""
    frames = _stacks(40, 3)
    _check_stem_forward(R, sms, frames, None)


def test_stem_forward_loops_over_stacks_bit_for_bit_and_fp64(R, sms):
    """n = 3 * (2 SMs) + 5, read through an idx that permutes the rows and repeats some: every CTA of the persistent
    kernel (grid 2 SMs) loops over three or four stacks, so the raw_full barrier's parity, the prefetch of the next
    stack into sRaw and the conv-row ring are reused across stacks.  Every stack bit for bit against stem_model's
    device restatement, and against fp64 through check_stem's per-element bounds."""
    n = 3 * 2 * sms + 5
    rows = n - 2 * sms                                          # the idx repeats 2 * SMs of the rows
    frames = _stacks(rows, 3)
    g = torch.Generator(device="cuda").manual_seed(11)
    perm = torch.randperm(rows, device="cuda", generator=g)
    idx = torch.cat([perm, perm[torch.randint(0, rows, (n - rows,), device="cuda", generator=g)]])
    _check_stem_forward(R, sms, frames, idx[torch.randperm(n, device="cuda", generator=g)].contiguous())


def _check_stem_forward(R, sms, frames, idx):
    n = len(frames) if idx is None else idx.numel()
    w = _weights(1)
    fr = torch.from_numpy(frames).cuda()
    pack = R.StemPack("cuda")
    pack.pack(w.cuda())
    pooled, amax = R.stem_fused(fr, idx, pack)
    pooled2, amax2 = R.stem_fused(fr, idx, pack)
    torch.cuda.synchronize()
    assert pooled.shape == (n, 16, 42, 42)
    assert torch.equal(pooled, pooled2) and torch.equal(amax, amax2)               # run to run
    q, scale = M.pack(w.numpy())
    assert np.array_equal(pack.scale.cpu().numpy(), scale)
    bq = pack.bq.cpu().numpy().reshape(4, 16, 12, 4)
    assert np.array_equal(bq[..., :3].reshape(4, 16, 36), q) and not bq[..., 3].any()
    want_p, want_a = M.forward_t(fr, idx, w.cuda())
    bad = ((pooled.view(torch.int32) != want_p.view(torch.int32)) | (amax != want_a)).flatten(1).any(1)
    print(f"[bits] stem forward n={n}, grid {min(n, 2 * sms)}: {int(bad.sum())} of {n} stacks differ")
    assert not bad.any(), f"stacks {bad.nonzero()[:8, 0].tolist()} differ from the device restatement"
    if idx is None:
        for lo in range(0, n, 8):                                               # the numpy loops in pieces (memory)
            want_p, want_a = M.pool(M.conv(frames[lo:lo + 8], w.numpy()))
            assert np.array_equal(pooled[lo:lo + 8].cpu().numpy(), want_p), lo
            assert np.array_equal(amax[lo:lo + 8].cpu().numpy(), want_a), lo
        # constant stacks: windows of interior conv rows all tie -> position 0; windows on the border never pick a
        # padded position (the conv output differs at the border: its patches reach into the zero padding)
        for k in (1, 2, 3):
            assert amax[k, :, 1:41, 1:41].max().item() == 0
            assert amax[k, :, 0].min().item() >= 3 and amax[k, :, :, 0].remainder(3).min().item() >= 1
    check_stem(f"stem forward n={n}", fr, idx, w.cuda(), pooled, amax)


def test_stem_wgrad_within_the_fp64_bound_and_deterministic(R):
    """n = 300 > SMs: the weight gradient's CTAs (grid = SMs) loop over two or three stacks each.  Within one fp32 ulp
    of stem_model's device restatement of the kernel's arithmetic, and against fp64 through check_stem_wgrad's
    per-element bound, alone and accumulated into an existing gradient."""
    n = 300                                                 # more stacks than SMs: several per CTA
    frames = _stacks(n, 5)
    w = _weights(2)
    fr = torch.from_numpy(frames).cuda()
    pack = R.StemPack("cuda")
    pack.pack(w.cuda())
    pooled, amax = R.stem_fused(fr, None, pack)
    g = torch.Generator(device="cuda").manual_seed(3)
    gp = torch.randn(n, 16, 42, 42, device="cuda", generator=g)
    gp[7] *= 1e-3                                           # a stack of small gradients: its own digit scale
    gp[8] *= 1e-33                                          # and one whose digit exponent clamps at 27
    dw = R.stem_wgrad(fr, None, gp, amax)
    dw2 = R.stem_wgrad(fr, None, gp, amax)
    acc = dw.clone()
    R.stem_wgrad(fr, None, gp, amax, out=acc, accumulate=True)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw2)
    want = M.wgrad_t(fr, None, gp, amax)
    d = M.ulps(dw, want)
    print(f"[bits] stem wgrad n={n}: {int((d > 0).sum())} of {d.numel()} elements one ulp from the restatement")
    assert d.max().item() <= 1
    assert M.ulps(acc, M.wgrad_t(fr, None, gp, amax, base=dw)).max().item() <= 1
    check_stem_wgrad(f"stem wgrad n={n}", fr, None, gp, amax, dw)
    check_stem_wgrad(f"stem wgrad n={n} accumulated", fr, None, gp, amax, acc, base=dw)
    assert (acc.double() - 2 * dw.double()).abs().max().item() <= 2 ** -22 * dw.abs().max().item()


def _rollout_cols(n, T, seed):
    state, a, mu, r, done, _ = atari_rollouts(n, T=T, actors=6, episode=(2 * T, 6 * T), p_done=0.3 / T, seed=seed)
    return [state, a, mu, r, done]


def test_stem_is_bit_identical_across_frame_sources(R):
    """Stack store rows, the dedup plane table, the staged coded pool and a bound slot (frame table) holding the same
    frames give the same pooled output, argmax and weight gradient, bit for bit."""
    from distributed_rl_b200.learner_common import time_major_rows
    from test_gpu_29_impala_frame_dedup import _buffers
    T, cap, B = 20, 64, 24
    cols = _rollout_cols(64, T, seed=9)
    stack = R.DeviceReplay(cap, R.impala_fields(T), "cuda:0")
    raw = R.RolloutDedupReplay(cap, 40 * cap, 1024, T=T)
    coded = R.RolloutDedupReplay(cap, 40 * cap, 1024, T=T, pool_bytes=(40 * cap + 1) * 7072)
    for st in (stack, raw, coded):
        st.push([torch.from_numpy(x) for x in cols], torch.ones(64))
        st.seed(31, 0)
    out = _buffers(B, T)
    raw.uniform_fetch(B, T, out)
    rows = out["rows"]
    t_idx = torch.arange(T + 1, device="cuda").view(T + 1, 1)
    staged = coded.alloc_staged(B)
    src_staged = coded.stage_frames(out["idx"], staged)
    staged_rows = time_major_rows(torch.arange(B, device="cuda"), t_idx)
    slot = stack.field_view("state").view(-1, 4, 84, 84)[rows].contiguous()    # a served slot: time-major rows
    table = torch.tensor([slot.data_ptr()], dtype=torch.int64, device="cuda")
    bound = R.BoundFrames(table, 0, rows.numel())
    sources = [(stack.field_view("state").view(-1, 4, 84, 84), rows), (raw.frame_source("state"), rows),
               (src_staged, staged_rows), (bound, None)]
    pack = R.StemPack("cuda")
    pack.pack(_weights(4).cuda())
    g = torch.Generator(device="cuda").manual_seed(5)
    gp = torch.randn(rows.numel(), 16, 42, 42, device="cuda", generator=g)
    res = []
    for frames, r in sources:
        p, a = R.stem_fused(frames, r, pack)
        res.append((p, a, R.stem_wgrad(frames, r, gp, a)))
    torch.cuda.synchronize()
    for k, (p, a, dw) in enumerate(res[1:], 1):
        assert torch.equal(p, res[0][0]) and torch.equal(a, res[0][1]) and torch.equal(dw, res[0][2]), k
    for st in (stack, raw, coded):
        st.close()


def _learner(B, T, N, memory=None, **kw):
    from distributed_rl_b200 import impala
    torch.manual_seed(0)
    cfg = dict(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0",
               MODEL=impala.resnet_small_model())
    cfg.update(kw)
    return impala.Learner(impala.ImpalaConfig(**cfg), start_replay=False, memory=memory)


def _snap(out):
    return {k: v.clone() for k, v in out.items()}


KEYS = ("vtarget", "advantage", "objActor", "criticLoss")


def test_fused_step_against_train_on_the_pytorch_stem(R):
    """The same draw: fused_step (stem on libb2rl) against train() of a FUSED_CONV1=False learner on the staged batch,
    which runs PyTorch's conv + max_pool2d on the fp32 frames (cuDNN in fp32: allow_tf32 off).  SGD, so that the
    post-step weights differ by lr times the gradients' difference: the stem's weight gradient through StemGathered
    lands in conv_1.weight.grad as PyTorch's does.  Each tensor's update agrees within 1e-3 of its largest element:
    room for fp32 reorderings and for the rare max-pool windows whose nearly tied values the two convolutions order
    differently."""
    B, T, N = 16, 20, 40
    sgd = {"name": "sgd", "lr": 0.05}
    E = _learner(B, T, N, OPTIM_INFO=sgd)
    P = _learner(B, T, N, OPTIM_INFO=sgd, FUSED_CONV1=False)
    w0 = [q.detach().clone() for q in E.model.parameters()]
    cols = _rollout_cols(N, T, seed=21)
    for L in (E, P):
        L.memory.push_arrays(*cols)
    for seed in (7, 8):                         # the second step runs on the stem weights re-packed after the first
        E.memory._rng.manual_seed(seed)
        o = _snap(E.fused_step())
        P.memory._rng.manual_seed(seed)
        sel = P.memory.draw(B)
        b = P.memory.store.gather(sel)
        P.train((b["state"].transpose(0, 1).contiguous(), b["action"].t().contiguous(), b["mu"].t().contiguous(),
                 b["reward"].t().contiguous(), b["done"]))
        torch.cuda.synchronize()
        for key in KEYS:
            u, v = o[key].double(), P.last[key].double()
            assert (u - v).abs().max().item() <= 1e-4 * max(1.0, v.abs().max().item()), (seed, key)
    assert hasattr(E, "_stem_pack") and not hasattr(P, "_stem_pack")      # P ran the PyTorch stem, E the fused one
    assert not torch.equal(P.model.module00.conv_1.weight, w0[0])          # the stem's weights took steps
    for (name, pe), pp, p0 in zip(E.model.named_parameters(), P.model.parameters(), w0):
        de, dp = pe.double() - p0.double(), pp.double() - p0.double()
        assert (de - dp).abs().max().item() <= 1e-3 * dp.abs().max().item(), name


def test_captured_step_equals_the_eager_step(R):
    from test_gpu_19_served_sequences import _same_params_and_state
    B, T, N = 16, 20, 48
    E, G = _learner(B, T, N), _learner(B, T, N)
    cols = _rollout_cols(N, T, seed=61)
    for L in (E, G):
        L.memory.push_arrays(*cols)
        L.memory.store.seed(13, 0)

    def eager():
        c = E.cfg
        s = E._drawn_state()
        E.memory.store.uniform_fetch(c.BATCHSIZE, c.UNROLL_STEP, s.cur)
        E._train_core(s.frames, s.cur["rows"], s.cur["action"], s.cur["mu"], s.cur["reward"], s.cur["done"], 0)
        return _snap(dict(E.last, idx=s.cur["idx"]))

    outs_e = [eager() for _ in range(4)][-1:]
    outs_g = [_snap(G.fused_step(use_graph=True))]
    for _ in range(2):
        outs_e.append(eager())
        outs_g.append(_snap(G.fused_step(use_graph=True)))
    torch.cuda.synchronize()
    assert G._graph is not None
    for oe, og in zip(outs_e, outs_g):
        for key in KEYS + ("idx",):
            assert torch.equal(oe[key], og[key]), key
    _same_params_and_state(E.mOptim, G.mOptim)


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "captured"])
def test_dedup_and_coded_stores_step_as_the_stack_store(R, use_graph):
    from test_gpu_19_served_sequences import _same_params_and_state
    B, T, N = 32, 20, 96
    kw = dict(FRAMES_PER_ROLLOUT=40.0, DEDUP_WINDOW=256)
    Ls = [_learner(B, T, N), _learner(B, T, N, FRAME_DEDUP=True, **kw),
          _learner(B, T, N, FRAME_DEDUP=True, STAGED_POOL_CODEC=True, **kw)]
    cols = _rollout_cols(N, T, seed=41)
    for L in Ls:
        L.memory.push_arrays(*cols)
        L.memory.store.seed(13, 0)
    for step in range(4):
        outs = []
        for L in Ls:
            L.memory._rng.manual_seed(100 + step)           # the eager draw's generator
            outs.append(_snap(L.fused_step(use_graph=use_graph)))
        torch.cuda.synchronize()
        for o in outs[1:]:
            for key in KEYS:
                assert torch.equal(outs[0][key], o[key]), (step, key)
    for L in Ls[1:]:
        _same_params_and_state(Ls[0].mOptim, L.mOptim)


def test_served_captured_step_equals_the_in_process_captured_step(R):
    """Slots filled by the served uniform fill from the same RNG state as the in-process draw hold the same rollouts:
    the bound step (3 eager warm-ups, the capture, replays) follows the in-process captured step bit for bit."""
    from test_gpu_19_served_sequences import _bind, _local_memory, _same_params_and_state
    from distributed_rl_b200.replay_server import ServeRing
    B, T, N, slots = 16, 20, 48, 6
    G = _learner(B, T, N)
    cols = _rollout_cols(N, T, seed=71)
    G.memory.push_arrays(*cols)
    st = G.memory.store
    ring = ServeRing.create(st, B, slots)
    try:
        st.seed(17, 0)
        for k in range(slots):
            ring.fill_uniform(st, k, 100 + k, T)
        torch.cuda.synchronize()
        S = _learner(B, T, 8, SERVED_FUSED_STEP=True, memory=_local_memory(ring))
        s = S._bound_state()
        served = []
        for k in range(slots):
            _bind(ring, k, R.impala_fields(T), s)
            served.append(_snap(S._bound_step()))
        st.seed(17, 0)
        local = [_snap(G.fused_step(use_graph=True))]           # draws 0..2 warm up, draw 3 is captured
        local += [_snap(G.fused_step(use_graph=True)) for _ in range(slots - 4)]
        torch.cuda.synchronize()
        assert S._graph is not None and G._graph is not None
        for k, o in enumerate(local):
            for key in KEYS:
                assert torch.equal(served[3 + k][key], o[key]), (k, key)
        _same_params_and_state(S.mOptim, G.mOptim)
    finally:
        torch.cuda.synchronize()
        ring.close()
