"""GPU tests of R2D2 on the IMPALA residual network (r2d2.resnet_model()): the two-network stem launch
(csrc/stem.cu b2rl_stem_fused_pair, R.stem_fused_pair) and the R2D2 learner's stem path.

The pair launch against two single-net launches (R.stem_fused) bit for bit, pooled values and the online net's argmax,
over every frame source R2D2 reads (stacks, strip windows, a strip dedup store's stride-1 plane table, a bound ring
slot), through an idx that permutes and repeats rows, at three or four stacks per CTA of the persistent kernel.  The
learner: the fused step against train() on the PyTorch stem over two Adam steps, with negative controls; the captured
step against the eager one; the served bound step against train() on the same slot, stacks and strips; and every
store form (strips, FRAME_DEDUP, HOST_FRAMES, HOST_POOL, POOL_CODEC) against a stack store."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from strip_dedup_model import player_sequences                  # noqa: E402

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


def _stream(n, T, seed):
    strips, a, r, h0, h1, nd, _ = player_sequences(n, T=T, actors=5, episode=(2 * T, 5 * T), seed=seed)
    p = (np.random.default_rng(seed + 100).random(n) + 0.01).astype(np.float32)
    return strips, a, r, h0, h1, nd, p


def _weights(seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(16, 4, 3, 3, generator=g) * scale).cuda()


# ---- the pair launch --------------------------------------------------------------------------------------------------
def test_pair_launch_equals_two_single_net_launches_on_every_source(R):
    """n = 3 * (2 SMs) + 5 rows (the pair kernel runs two CTAs per SM, so each CTA loops over three or four stacks),
    drawn through an idx that permutes the rows and repeats some, from four sources holding the same windows: stacks,
    the windows of frame strips, a StripDedupReplay's stride-1 plane table and a BoundFrames table entry.  Each net's
    pooled output is bit for bit stem_fused's with that net's pack, net 0's argmax is stem_fused's, and the pooled
    outputs are the same with and without the argmax, on every source and across two runs."""
    from test_gpu_27_r2d2_frame_dedup import _stores
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    T, cap = 80, 24
    plain, dedup = _stores(R, 24, cap, T, seed=61)
    win = R.strip_windows(plain.field_view("state"))
    n = 3 * 2 * sms + 5
    g = torch.Generator(device="cuda").manual_seed(3)
    perm = torch.randperm(win.shape[0], device="cuda", generator=g)[:n - 2 * sms]
    idx = torch.cat([perm, perm[torch.randint(0, perm.numel(), (2 * sms,), device="cuda", generator=g)]])
    idx = idx[torch.randperm(n, device="cuda", generator=g)].contiguous()
    stacks = win[torch.arange(win.shape[0], device="cuda")].contiguous()
    table = torch.tensor([plain.field_view("state").data_ptr()], dtype=torch.int64, device="cuda")
    bound = R.BoundFrames(table, 0, win.shape[0], R.FRAME_BYTES)
    sources = {"stacks": stacks, "strip windows": win, "plane table": dedup.frame_source("state"), "bound": bound}
    assert sources["plane table"].plane_stride == 1
    on, tg = R.StemPack("cuda"), R.StemPack("cuda")
    on.pack(_weights(1))
    tg.pack(_weights(2, 0.05))
    pair = R.stem_pack_pair("cuda")
    pair[0].pack(_weights(1))
    pair[1].pack(_weights(2, 0.05))
    want_on, want_a = R.stem_fused(stacks, idx, on)
    want_tg, _ = R.stem_fused(stacks, idx, tg)
    for name, src in sources.items():
        for packs in ((on, tg), pair):                      # copied side by side, and read in place
            p_on, p_tg, a = R.stem_fused_pair(src, idx, *packs)
            q_on, q_tg, none = R.stem_fused_pair(src, idx, *packs, argmax=False)
            r_on, r_tg, a2 = R.stem_fused_pair(src, idx, *packs)
            torch.cuda.synchronize()
            assert none is None
            for got, want in ((p_on, want_on), (p_tg, want_tg), (a, want_a), (q_on, want_on), (q_tg, want_tg),
                              (r_on, p_on), (r_tg, p_tg), (a2, a)):
                assert torch.equal(got, want), name
    assert not torch.equal(want_on, want_tg)
    for st in (plain, dedup):
        st.close()


def test_pair_entry_point_refuses_bad_arguments(R):
    from distributed_rl_b200 import _lib
    lib = _lib.load()
    frames = torch.zeros(2, 4, 84, 84, dtype=torch.uint8, device="cuda")
    src = R._frame_source(frames)
    bq = torch.zeros(2 * 3072 + 16, dtype=torch.int8, device="cuda")
    sc = torch.zeros(32, device="cuda")
    out = torch.empty(2, 2, 16, 42, 42, device="cuda")
    assert lib.b2rl_stem_fused_pair(src, None, 2, bq.data_ptr() + 4, sc.data_ptr(), out.data_ptr(), None, None) == -1
    assert b"16-byte" in lib.b2rl_last_error()
    assert lib.b2rl_stem_fused_pair(src, None, 2, bq.data_ptr(), sc.data_ptr(), None, None, None) == -1
    assert lib.b2rl_stem_fused_pair(src, None, 0, None, None, None, None, None) == 0       # nothing to do


# ---- the learner ------------------------------------------------------------------------------------------------------
def _learner(memory=None, **kw):
    from distributed_rl_b200 import r2d2
    torch.manual_seed(0)
    cfg = dict(BATCHSIZE=8, FIXED_TRAJECTORY=80, MEM=20, REPLAY_MEMORY_LEN=32, LEARNER_DEVICE="cuda:0",
               MODEL=r2d2.resnet_model())
    cfg.update(kw)
    return r2d2.Learner(r2d2.R2D2Config(**cfg), start_replay=False, memory=memory)


def _push(L, cols, strips: bool):
    from distributed_rl_b200 import replay as R
    s, a, r, h0, h1, nd, p = cols
    if not strips:
        s = R.strip_stacks(torch.from_numpy(s)).contiguous().numpy()
    L.memory.push_arrays(s, a, r, h0, h1, nd, p)


def _recording_grads(L):
    """Record every parameter's gradient before each optimizer step (step() zeroes them)."""
    from distributed_rl_b200 import r2d2
    L.grads = []

    def step():
        L.grads.append([q.grad.clone() for q in L.model.parameters()])
        return r2d2.Learner.step(L)
    L.step = step


# The fused step against train() on the PyTorch stem, the same batch for both, two Adam steps.  Both learners run the
# same 3xTF32 heads, and TF32 is off here, so the PyTorch learner's stem, residual blocks and LSTM run in fp32 on cuDNN.
# The two differ in the stem: the kernel's exact integer digit sums recombined in fp32 against cuDNN's fp32 conv (within
# 2e-6 relative, tests/test_impala_resnet_cpu.py), which also lets a nearly tied max-pool window pick another position
# and route its gradient there.  The residual blocks and the LSTM carry that to the loss and the priorities, and Adam
# carries the stem's weight-gradient difference into every step's update of elements whose second moment is small.
# Each figure is a relative error, max |fused - pytorch| / max |pytorch| over the two steps (params: of the change from
# the initial weights).  Measured on an H100 80GB HBM3: prio 7.6e-8, loss 1.6e-7, stem grad 5.3e-4, params 2.2e-3.
# The bounds leave 130x, 64x, 19x and 9x room over those; the negative controls below give stem grad 0.65-1.11 and
# params 1.24-1.37, 30x or more above the bounds.
TOL = {"prio": 1e-5, "loss": 1e-5, "stem grad": 1e-2, "params": 2e-2}


def _step_errors(F, P, batches, bad=None, monkeypatch=None):
    """Relative errors of the fused learner F against the PyTorch learner P over `batches`; `bad` replaces
    R.stem_fused_pair inside F's steps (a negative control)."""
    from distributed_rl_b200 import replay as R
    w0 = [q.detach().clone() for q in P.model.parameters()]
    err = dict.fromkeys(TOL, 0.0)

    def rel(u, v):
        return (u.double() - v.double()).abs().max().item() / max(v.double().abs().max().item(), 1e-30)
    for batch in batches:
        if bad is not None:
            monkeypatch.setattr(R, "stem_fused_pair", bad)
        info_f, prio_f, _ = F.train(batch)
        if bad is not None:
            monkeypatch.undo()
        info_p, prio_p, _ = P.train(batch)
        torch.cuda.synchronize()
        err["prio"] = max(err["prio"], rel(prio_f, prio_p))
        err["loss"] = max(err["loss"], rel(info_f["loss"], info_p["loss"]))
        err["stem grad"] = max(err["stem grad"], rel(F.grads[-1][0], P.grads[-1][0]))
    for qf, qp, q0 in zip(F.model.parameters(), P.model.parameters(), w0):
        err["params"] = max(err["params"], rel(qf - q0, qp - q0))
    return err


def _pytorch_pair():
    F, P = _learner(), _learner(FUSED_CONV1=False)
    cols = _stream(32, 80, seed=71)
    for L in (F, P):
        _push(L, cols, strips=False)
        _recording_grads(L)
    assert F.model.first_stem_node() == "module00"
    F.memory.store.seed(5, 0)
    batches = []
    for _ in range(2):
        F.memory.buffer(1)
        batches.append(F.memory.deque.pop())
    assert batches[0][1].dtype == torch.uint8
    return F, P, batches


def test_fused_step_against_train_on_the_pytorch_stem(R):
    F, P, batches = _pytorch_pair()
    err = _step_errors(F, P, batches)
    print("[r2d2 resnet] fused vs PyTorch, relative errors: " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert hasattr(F, "_stem_packs") and not hasattr(P, "_stem_packs")   # F ran the pair kernel, P PyTorch's stem
    assert F.grads[0][0].abs().max().item() > 0
    for k, tol in TOL.items():
        assert err[k] <= tol, (k, err[k])


@pytest.mark.parametrize("control", ["target pooled to the online net", "argmax dropped"])
def test_negative_controls_fail_the_step_comparison(R, monkeypatch, control):
    real = R.stem_fused_pair

    def bad(frames, idx, pack_online, pack_target, argmax=True, out=None):
        p_on, p_tg, a = real(frames, idx, pack_online, pack_target, argmax, out)
        if not argmax:
            return p_on, p_tg, a
        if control == "argmax dropped":
            return p_on, p_tg, torch.zeros_like(a)
        return p_tg, p_tg, a
    F, P, batches = _pytorch_pair()
    err = _step_errors(F, P, batches, bad=bad, monkeypatch=monkeypatch)
    print(f"[r2d2 resnet] negative control ({control}): " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert any(err[k] > 30 * TOL[k] for k in TOL), err


def _same_params_and_state(opt_a, opt_b):
    from test_gpu_19_served_sequences import _same_params_and_state as same
    same(opt_a, opt_b)


def test_captured_step_equals_the_eager_step(R):
    from test_gpu_19_served_sequences import _fill
    N = 32
    G, E = _learner(), _learner()
    for L in (G, E):
        _fill(L.memory.store, N, 51)
        L.memory.store.seed(13, 0)
    outs_e = [E.fused_step() for _ in range(4)][-1:]
    outs_g = [{k: v.clone() for k, v in G.fused_step(use_graph=True).items()}]
    assert G._graph is not None and E._graph is None
    for _ in range(2):
        outs_e.append({k: v.clone() for k, v in E.fused_step().items()})
        outs_g.append({k: v.clone() for k, v in G.fused_step(use_graph=True).items()})
    torch.cuda.synchronize()
    for oe, og in zip(outs_e, outs_g):
        for key in ("idx", "prio", "scalars", "p_norm"):
            assert torch.equal(oe[key], og[key]), key
    assert len({tuple(o["idx"].tolist()) for o in outs_g}) > 1
    assert torch.equal(E.memory.store.priorities(0, N), G.memory.store.priorities(0, N))
    _same_params_and_state(E.optim, G.optim)


@pytest.mark.parametrize("strip", [False, True], ids=["stacks", "strips"])
def test_served_bound_step_equals_train_on_the_slot(R, strip):
    """The bound step (3 eager warm-ups, the capture, replays after rebinds) reads the slot through the BoundFrames
    entry (frame strips: windows 7 056 bytes apart); train() runs on a copy of the same slot."""
    from test_gpu_19_served_sequences import _bind, _local_memory, _take
    from distributed_rl_b200.replay_server import KINDS, ServeRing
    B, T, N, slots = 8, 80, 40, 6
    fields = R.r2d2_fields(T, strip=strip)
    st = R.DeviceReplay(N, fields, "cuda:0")
    s_, a, r, h0, h1, nd, p = _stream(N, T, seed=81)
    if not strip:
        s_ = R.strip_stacks(torch.from_numpy(s_)).contiguous().numpy()
    st.push([torch.from_numpy(x) for x in (s_, a, r, h0, h1, nd)], torch.from_numpy(p))
    ring = ServeRing.create(st, B, slots)
    try:
        st.seed(7, 0)
        for k in range(slots):
            ring.fill(st, k, 100 + k, 0.4)
        A = _learner(memory=_local_memory(ring), FRAME_STRIP=strip, SERVED_FUSED_STEP=True, REPLAY_MEMORY_LEN=8)
        Bl = _learner(FRAME_STRIP=strip, REPLAY_MEMORY_LEN=8)
        s = A._state()
        assert s.frames["state"].row_stride == (R.FRAME_BYTES if strip else R.FRAME_STACK_BYTES)
        for k in range(slots):
            _bind(ring, k, fields, s)
            out = A._bound_step()
            hdr, idx, w, b = _take(ring, k, fields, False)
            info, prio, idx_b = Bl.train(KINDS["r2d2"].batch(b, w, idx))
            torch.cuda.synchronize()
            assert (A._graph is not None) == (k >= A.BOUND_WARMUP), k
            assert torch.equal(out["idx"], idx_b) and torch.equal(out["prio"], prio), k
            assert torch.equal(out["scalars"][0], info["loss"]) and torch.equal(out["p_norm"], info["p_norm"]), k
            _same_params_and_state(A.optim, Bl.optim)
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


STORES = {"strips": dict(FRAME_STRIP=True),
          "FRAME_DEDUP": dict(FRAME_DEDUP=True, FRAMES_PER_SEQUENCE=120, DEDUP_WINDOW=1024),
          "HOST_FRAMES": dict(FRAME_STRIP=True, HOST_FRAMES=True),
          "HOST_POOL": dict(FRAME_DEDUP=True, HOST_POOL=True, FRAMES_PER_SEQUENCE=120, DEDUP_WINDOW=1024),
          "POOL_CODEC": dict(FRAME_DEDUP=True, POOL_CODEC=True, FRAMES_PER_SEQUENCE=120, DEDUP_WINDOW=1024)}


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "captured"])
def test_every_store_steps_as_the_stack_store(R, use_graph):
    """The same sequences in a stack store and in each other store form, the trees seeded alike: the fused steps are
    bit for bit the same (the stem reads stacks, strip windows, the plane table, or the staging buffer the host and
    coded stores fill)."""
    N = 32
    cols = _stream(N, 80, seed=91)
    Ls = {"stacks": _learner()}
    Ls.update({name: _learner(**kw) for name, kw in STORES.items()})
    for name, L in Ls.items():
        _push(L, cols, strips=name != "stacks")
        L.memory.store.seed(13, 0)
    for step in range(3):
        outs = {name: L.fused_step(use_graph=use_graph) for name, L in Ls.items()}
        torch.cuda.synchronize()
        for name, o in outs.items():
            for key in ("idx", "prio", "scalars", "p_norm"):
                assert torch.equal(outs["stacks"][key], o[key]), (step, name, key)
    for name, L in Ls.items():
        assert (L._graph is not None) == use_graph, name
        _same_params_and_state(Ls["stacks"].optim, L.optim)
