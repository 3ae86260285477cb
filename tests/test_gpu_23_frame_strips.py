"""GPU tests of R2D2 frame strips (R2D2Config.FRAME_STRIP): strips and stacks give the same bits.

Kernels: conv_1 forward and weight gradient over the windows of frame strips (rows 7 056 bytes apart) against the
same kernels over the materialised stacks, for direct and table sources, time-major rows with repeated slots, ReLU
on and off, one and two networks, 32 and 16 channels, the last window of the allocation and a weight gradient split
over two launches.  Learner: train(), the captured in-process fused_step and the captured served step on strips
against stacks, a two-process run, the reference-format ingest, and a 100 000-sequence strip replay on an 80 GB card."""
import multiprocessing as mp
import pickle
import time

import numpy as np
import pytest

from shared_redis import RedisManager, Shim

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(autouse=True)
def _deterministic():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    b = torch.backends
    saved = (b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32)
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = True, False, False, False
    yield
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = saved


def _strips(n, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n, T + 3, 84, 84), dtype=torch.uint8, device="cuda", generator=g)


def _pack(n_nets, c_out, seed):
    from distributed_rl_b200 import replay as R
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = R.Conv1Pack(n_nets, "cuda", c_out)
    for net in range(n_nets):
        p.pack(net, torch.randn(c_out, 4, 8, 8, device="cuda", generator=g) * 0.05)
    return p


def _gy(n, c_out, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, c_out, 20, 20, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)


def _sources(strips):
    """-> (window view, the materialised stacks of the same rows, a BoundFrames over the strips, its table)."""
    from distributed_rl_b200 import replay as R
    win = R.strip_windows(strips)
    table = torch.tensor([0, strips.data_ptr()], dtype=torch.int64, device="cuda")
    return win, win.contiguous(), R.BoundFrames(table, 1, win.shape[0], R.FRAME_BYTES), table


@pytest.mark.parametrize("c_out", [32, 16])
@pytest.mark.parametrize("n_nets", [1, 2])
@pytest.mark.parametrize("relu", [False, True])
def test_conv1_on_windows_equals_conv1_on_stacks(relu, n_nets, c_out):
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.learner_common import time_major_rows
    T, S = 80, 9
    win, stacks, bound, _ = _sources(_strips(S, T, 1))
    assert win.shape[0] == S * (T + 3) - 3 and stacks.stride(0) == R.FRAME_STACK_BYTES
    pack = _pack(n_nets, c_out, 2)
    seq = torch.tensor([4, 0, 8, 4, 2, 8], device="cuda")                       # repeated slots, the last sequence
    rows = time_major_rows(seq, torch.arange(T, device="cuda").view(T, 1), T + 3)
    last = torch.tensor([win.shape[0] - 1, 0, win.shape[0] - 1], device="cuda")  # the last window of the allocation
    for idx in (rows, last, None):
        want = R.conv1_fused(stacks, idx, pack, relu=relu)
        for src in (win, bound):
            for a, b in zip(want, R.conv1_fused(src, idx, pack, relu=relu)):
                assert torch.equal(a, b)
        n = win.shape[0] if idx is None else idx.numel()
        gy = _gy(n, c_out, 3)
        y = want[0] if relu else None
        gw = R.conv1_wgrad(stacks, idx, gy, relu_y=y)
        for src in (win, bound):
            assert torch.equal(gw, R.conv1_wgrad(src, idx, gy, relu_y=y))
            acc = torch.ones_like(gw)
            R.conv1_wgrad(src, idx, gy, out=acc, accumulate=True, relu_y=y)
            ref = torch.ones_like(gw)
            R.conv1_wgrad(stacks, idx, gy, out=ref, accumulate=True, relu_y=y)
            assert torch.equal(acc, ref)


@pytest.mark.parametrize("accumulate", [False, True])
def test_weight_gradient_over_windows_split_over_two_launches(accumulate):
    """n = SMs * 160 + 257 windows without idx: the second launch starts off * 7 056 bytes into the strips."""
    from distributed_rl_b200 import replay as R
    per_launch = torch.cuda.get_device_properties(0).multi_processor_count * 160
    n = per_launch + 257
    T = 80
    S = (n + 3 + T + 2) // (T + 3)
    win, stacks, bound, _ = _sources(_strips(S, T, 6))
    win, stacks = win[:n], stacks[:n]
    bound = R.BoundFrames(bound.table, bound.entry, n, R.FRAME_BYTES)
    gy = _gy(n, 32, 7)
    y = torch.relu(_gy(n, 32, 8))
    outs = []
    for src in (stacks, win, bound):
        out = torch.full((32, 4, 8, 8), 0.25, device="cuda")
        outs.append(R.conv1_wgrad(src, None, gy, out=out, accumulate=accumulate, relu_y=y))
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    part = R.conv1_wgrad(win[:per_launch], None, gy[:per_launch], relu_y=y[:per_launch])
    assert not torch.equal(R.conv1_wgrad(win, None, gy, relu_y=y), part)      # the second launch's rows count
    del win, stacks, bound, gy, y
    torch.cuda.empty_cache()


# ---- the learner ----------------------------------------------------------------------------------------------------
def _sliding_batch(n, T, seed):
    """n sequences that slide: (strips on the host, stacks on the host, action, reward, h0, h1, notdone, priority)."""
    rng = np.random.default_rng(seed)
    strips = rng.integers(0, 256, (n, T + 3, 84, 84), dtype=np.uint8)
    stacks = np.lib.stride_tricks.as_strided(strips, (n, T, 4, 84, 84),
                                             (strips.strides[0],) + strips.strides[1:2] * 2 + strips.strides[2:]).copy()
    return (strips, stacks, rng.integers(0, 6, (n, T)).astype(np.int32), rng.standard_normal((n, T)).astype(np.float32),
            (0.1 * rng.standard_normal((n, 512))).astype(np.float32),
            (0.1 * rng.standard_normal((n, 512))).astype(np.float32),
            (rng.random(n) > 0.1).astype(np.float32), (rng.random(n) + 0.05).astype(np.float32))


def _same_params_and_state(opt_a, opt_b):
    for pa, pb in zip(opt_a.param_groups[0]["params"], opt_b.param_groups[0]["params"]):
        assert torch.equal(pa, pb)
        sa, sb = opt_a.state[pa], opt_b.state[pb]
        assert sa.keys() == sb.keys()
        for key in sa:
            assert torch.equal(sa[key], sb[key]), key


def _pair(**kw):
    """Two learners of the same weights and config, one storing strips and one stacks."""
    from distributed_rl_b200 import r2d2
    out = []
    for strip in (True, False):
        torch.manual_seed(0)
        out.append(r2d2.Learner(r2d2.R2D2Config(**kw, FRAME_STRIP=strip), start_replay=False))
    return out


def _push(L, batch, strip_input=True):
    strips, stacks, *rest = batch
    L.memory.push_arrays(strips if (strip_input and L.cfg.FRAME_STRIP) else stacks, *rest)


def test_train_on_strips_equals_train_on_stacks():
    B, T, N = 8, 80, 24
    S, K = _pair(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0")
    batch = _sliding_batch(N, T, 11)
    _push(S, batch, strip_input=False)                  # stacks encoded on ingest
    _push(K, batch)
    assert S.memory.store.field_view("state").shape == (N, T + 3, 84, 84)
    for L in (S, K):
        L.memory.store.seed(5, 0)
    for step in range(3):
        bs, bk = S.memory.sample(), K.memory.sample()
        assert bs[1].stride()[1:] == (7056, 7056, 84, 1) and torch.equal(bs[1], bk[1])     # the stack view
        info_s, prio_s, idx_s = S.train(bs)
        info_k, prio_k, idx_k = K.train(bk)
        assert torch.equal(idx_s, idx_k) and torch.equal(prio_s, prio_k), step
        for key in ("loss", "mean_value", "p_norm"):
            assert torch.equal(info_s[key], info_k[key]), key
        S.memory.update(idx_s, prio_s)
        K.memory.update(idx_k, prio_k)
        _same_params_and_state(S.optim, K.optim)


def test_captured_fused_step_on_strips_equals_stacks_while_ingest_wraps():
    B, T, N = 8, 80, 32
    S, K = _pair(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0")
    for L in (S, K):
        _push(L, _sliding_batch(N, T, 21))
        L.memory.store.seed(13, 0)
    for step in range(6):
        if step in (2, 4):                              # ingests that wrap the ring head between replays
            b = _sliding_batch(20, T, 30 + step)
            for L in (S, K):
                _push(L, b)
        os_, ok = S.fused_step(use_graph=True), K.fused_step(use_graph=True)
        torch.cuda.synchronize()
        for key in ("idx", "prio", "scalars", "p_norm"):
            assert torch.equal(os_[key], ok[key]), (step, key)
    assert S._graph is not None and K._graph is not None
    assert torch.equal(S.memory.store.priorities(0, N), K.memory.store.priorities(0, N))
    _same_params_and_state(S.optim, K.optim)


def test_push_records_of_reference_format_sequences():
    from fake_redis import FakeRedis
    from test_frame_strips_cpu import _records
    from distributed_rl_b200 import r2d2, wire
    T, n = 80, 6
    strips, stacks, *_ = _sliding_batch(n, T, 41)
    conn = FakeRedis()
    conn.rpush("experience", *_records(stacks))
    rp = r2d2.Replay(r2d2.R2D2Config(BATCHSIZE=n, FIXED_TRAJECTORY=T, REPLAY_MEMORY_LEN=n, FRAME_STRIP=True,
                                     LEARNER_DEVICE="cuda:0"))
    rp.push_records(wire.drain(conn, "experience"))
    assert torch.equal(rp.store.field_view("state").cpu(), torch.from_numpy(strips))
    rp.store.seed(1, 0)
    rp.buffer(1)
    (h0, h1), s, a, r, nd, w, idx = rp.deque.pop()
    assert s.shape == (n, T, 4, 84, 84)
    assert torch.equal(s.cpu(), torch.from_numpy(stacks[idx.cpu().numpy()]))
    rp.store.close()


SLOTS = 6


def test_served_captured_step_on_strips_equals_train_on_the_slot():
    from test_gpu_19_served_sequences import _bind, _local_memory, _take
    from distributed_rl_b200 import r2d2, replay as R
    from distributed_rl_b200.replay_server import KINDS, ServeRing
    B, T, N = 8, 80, 40
    cfg = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=8, LEARNER_DEVICE="cuda:0", FRAME_STRIP=True)
    fields = R.r2d2_fields(T, strip=True)
    st = R.DeviceReplay(N, fields, "cuda:0")
    strips, stacks, a, r, h0, h1, nd, p = _sliding_batch(N, T, 51)
    st.push([strips, a, r, h0, h1, nd], p)
    ring = ServeRing.create(st, B, SLOTS)
    try:
        st.seed(7, 0)
        for k in range(SLOTS):
            ring.fill(st, k, 100 + k, 0.4)
        torch.manual_seed(0)
        A = r2d2.Learner(r2d2.R2D2Config(**cfg, SERVED_FUSED_STEP=True), start_replay=False, memory=_local_memory(ring))
        torch.manual_seed(0)
        Bl = r2d2.Learner(r2d2.R2D2Config(**dict(cfg, FRAME_STRIP=False)), start_replay=False)
        s = A._state()
        assert s.frames["state"].row_stride == 7056 and s.frames["state"].rows == B * (T + 3) - 3
        for k in range(SLOTS):
            _bind(ring, k, fields, s)
            out = A._bound_step()
            hdr, idx, w, b = _take(ring, k, fields, False)
            batch = KINDS["r2d2"].batch(b, w, idx)
            batch[1] = batch[1].contiguous()                       # the stack learner gets materialised stacks
            info, prio, idx_b = Bl.train(batch)
            torch.cuda.synchronize()
            assert (A._graph is not None) == (k >= A.BOUND_WARMUP), k
            assert torch.equal(out["idx"], idx_b) and torch.equal(out["prio"], prio), k
            assert torch.equal(out["scalars"][0], info["loss"]) and torch.equal(out["p_norm"], info["p_norm"]), k
            _same_params_and_state(A.optim, Bl.optim)
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


def test_two_process_served_captured_step_with_strips():
    from test_frame_strips_cpu import _records
    from test_gpu_19_served_sequences import _server_main
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200 import replay_server as RS
    N, B, T, steps = 40, 4, 80, 8
    base = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, REPLAY_MEMORY_LEN=64, BUFFER_SIZE=16, LEARNER_DEVICE="cuda:0",
                FRAME_STRIP=True)
    ctx = mp.get_context("spawn")
    mgr = RedisManager(ctx=ctx)
    mgr.start()
    child, stop, client = None, ctx.Event(), None
    try:
        proxy = mgr.Redis()
        conn = Shim(proxy)
        out = ctx.Queue()
        child = ctx.Process(target=_server_main, args=("r2d2", proxy, base, stop, out))
        child.start()
        _, stacks, *_ = _sliding_batch(N, T, 61)
        conn.rpush("experience", *_records(stacks))
        client = RS.DeviceReplayClient(r2d2.R2D2Config(**base), conn, timeout=180.0)
        assert client.ring.layout.field_bytes[0] == (T + 3) * 7056
        torch.manual_seed(0)
        L = r2d2.Learner(r2d2.R2D2Config(**base, SERVED_FUSED_STEP=True), connect=conn, start_replay=False,
                         memory=client)
        assert L.run(max_steps=steps, log_every=100) == steps
        torch.cuda.synchronize()
        assert L._graph is not None
        assert all(torch.isfinite(p).all() for p in L.model.parameters())
        client.close()
        client = None
        stop.set()
        _, freed = out.get(timeout=120)
        assert freed
    finally:
        stop.set()
        if client is not None:
            client.close()
        if child is not None:
            child.join(timeout=60)
            if child.is_alive():
                child.terminate()
                child.join()
        mgr.shutdown()


def test_a_100k_sequence_strip_replay_fits_and_steps():
    """10^5 strip sequences (59.0 GB) on one 80 GB card: allocated, hash-filled, built, stepped by the captured
    fused_step.  Stacks would need 226 GB."""
    from distributed_rl_b200 import r2d2, replay as R
    total = torch.cuda.get_device_properties(0).total_memory
    if total < 75 * 2 ** 30:
        pytest.skip(f"needs an 80 GB card ({total / 2 ** 30:.0f} GiB)")
    N, B, T = 100_000, 64, 80
    per_seq = sum(f.nbytes for f in R.r2d2_fields(T, strip=True))
    assert per_seq == 590_388 and N * per_seq < 59.1e9
    torch.manual_seed(0)
    L = r2d2.Learner(r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, FRAME_STRIP=True,
                                     LEARNER_DEVICE="cuda:0"), start_replay=False)
    st = L.memory.store
    st.fill_hash(N, seed=3)
    g = torch.Generator(device="cuda").manual_seed(3)
    st.field_view("action").random_(0, 6, generator=g)
    st.field_view("reward").normal_(generator=g)
    for name in ("h0", "h1"):
        st.field_view(name).normal_(0.0, 0.1, generator=g)
    st.field_view("notdone").bernoulli_(0.9, generator=g)
    st.build(torch.rand(N, device="cuda", generator=g) + 0.05)
    st.seed(1, 0)
    outs = [L.fused_step(use_graph=True) for _ in range(3)]
    torch.cuda.synchronize()
    assert L._graph is not None and torch.isfinite(outs[-1]["prio"]).all()
    assert int(outs[-1]["idx"].max()) < N
    del L, st
    torch.cuda.empty_cache()
