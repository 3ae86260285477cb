"""GPU tests of R2D2 host frames (R2D2Config.HOST_FRAMES, DeviceReplay(host_fields=...)): a replay whose `state`
rows live in pinned host memory gives the bits of the same replay in HBM.

Gather: the host-row kernel alone at rows of 16 B to a stack sequence against index_select on the CPU view (clamped,
repeated and last rows, n = 1 and n = 64), and a host store against an HBM store fed by each ingest path (push from
pageable, pinned and device rows, push_begin / push_commit, ingest_pipelined, fill_hash) across a ring wrap.
Learner: train() on Replay.buffer() batches, the eager and the captured fused_step (also while push_arrays wraps the
ring between replays), strips and stacks.  Served: ring slots filled from a host store, and the served captured step
on them.  Placement: the host field is pinned host memory, a 4 096-sequence host-strip store takes no frame memory on
the device, and the refusals come before any launch.  At most 2.4 GB is pinned at a time."""
import ctypes

import numpy as np
import pytest

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
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _pair_of_stores(capacity, fields):
    from distributed_rl_b200 import replay as R
    return (R.DeviceReplay(capacity, fields, "cuda:0", host_fields=("state",)),
            R.DeviceReplay(capacity, fields, "cuda:0"))


# ---- the host-row gather ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row_bytes", [16, 1024, 585_648, 2_257_920])
def test_host_row_gather_equals_index_select(row_bytes):
    from distributed_rl_b200 import replay as R
    cap = max(8, min(96, (1 << 28) // row_bytes))
    st = R.DeviceReplay(cap, (R.Field("state", torch.uint8, (row_bytes,)),), "cuda:0", host_fields=("state",))
    st.fill_hash(cap, seed=row_bytes)
    torch.cuda.synchronize()
    view = st.field_view("state")
    assert view.device.type == "cpu" and view.shape == (cap, row_bytes)
    g = torch.Generator().manual_seed(row_bytes)
    for idx in (torch.randint(0, cap, (64,), generator=g), torch.tensor([cap - 1]),
                torch.tensor([cap - 1, 0, 3, 3, cap - 1, -5, cap + 7, 1])):
        out = st.gather(idx.cuda())["state"]
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), view.index_select(0, idx.clamp(0, cap - 1))), idx
    st.close()


# ---- host store against HBM store, per ingest path --------------------------------------------------------------------
def _records(fields, n, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for f in fields:
        if f.dtype == torch.uint8:
            out.append(torch.randint(0, 256, (n,) + tuple(f.shape), dtype=torch.uint8, generator=g))
        elif f.dtype == torch.int32:
            out.append(torch.randint(0, 6, (n,) + tuple(f.shape), dtype=torch.int32, generator=g))
        else:
            out.append(torch.randn((n,) + tuple(f.shape), generator=g))
    return out, torch.rand(n, generator=g) + 0.05


def _ingest(st, path, batches):
    from distributed_rl_b200 import hostmem
    for k, (cols, p) in enumerate(batches):
        if path == "push":                               # pageable, pinned, device rows in turn
            src = [c.numpy() for c in cols] if k % 3 == 0 else \
                [hostmem.pinned_like(c, st.device) for c in cols] if k % 3 == 1 else [c.cuda() for c in cols]
            st.push(src, p)
        elif path == "push_begin":
            pinned = [hostmem.pinned_like(c, st.device) for c in cols]
            st.push_begin(pinned, len(p))
            st.push_commit(p.cuda())
        elif path == "ingest_pipelined":
            pinned = [hostmem.pinned_like(c, st.device) for c in cols]
            st.ingest_pipelined(pinned, hostmem.pinned_like(p, st.device))
            torch.cuda.synchronize()                     # the pinned staging is dropped at the next iteration
        else:
            raise AssertionError(path)
    if path == "ingest_pipelined":
        st.ingest_pipelined(None)


@pytest.mark.parametrize("strip", [True, False])
@pytest.mark.parametrize("path", ["push", "push_begin", "ingest_pipelined", "fill_hash"])
def test_gather_from_a_host_store_equals_an_hbm_store(path, strip):
    from distributed_rl_b200 import replay as R
    N = 10
    fields = R.r2d2_fields(80, strip=strip)
    H, D = _pair_of_stores(N, fields)
    if path == "fill_hash":
        for st in (H, D):
            st.fill_hash(N, seed=77)
            st.build(torch.rand(N, device="cuda", generator=torch.Generator("cuda").manual_seed(1)) + 0.05)
    else:
        batches = [_records(fields, n, 10 + k) for k, n in enumerate((6, 7, 5))]     # wraps the ring twice
        for st in (H, D):
            _ingest(st, path, batches)
    torch.cuda.synchronize()
    assert len(H) == len(D) == N and H.head == D.head
    assert torch.equal(H.field_view("state"), D.field_view("state").cpu())
    g = torch.Generator().manual_seed(3)
    for idx in (torch.randint(0, N, (64,), generator=g), torch.tensor([N - 1]), torch.tensor([N - 1, 0, N - 1, 4])):
        a, b = H.gather(idx.cuda()), D.gather(idx.cuda())
        torch.cuda.synchronize()
        for f in fields:                                 # bit views: hash-filled floats include NaNs
            assert torch.equal(a[f.name].view(torch.uint8), b[f.name].view(torch.uint8)), (f.name, idx)
    for st in (H, D):
        st.seed(9, 0)
    assert torch.equal(H.sample(16)[0], D.sample(16)[0])
    H.close()
    D.close()


# ---- the learner ------------------------------------------------------------------------------------------------------
def _learners(strip, **kw):
    """Two learners of the same weights: frames in host memory, frames in HBM."""
    from distributed_rl_b200 import r2d2
    out = []
    for host in (True, False):
        torch.manual_seed(0)
        out.append(r2d2.Learner(r2d2.R2D2Config(**kw, FRAME_STRIP=strip, HOST_FRAMES=host), start_replay=False))
    return out


def _push(L, batch):
    from test_gpu_23_frame_strips import _push as push
    push(L, batch)


def _same(H, D, outs_h, outs_d, step):
    from test_gpu_23_frame_strips import _same_params_and_state
    for key in ("idx", "prio", "scalars", "p_norm"):
        assert torch.equal(outs_h[key], outs_d[key]), (step, key)
    _same_params_and_state(H.optim, D.optim)


@pytest.mark.parametrize("strip", [True, False])
def test_train_and_eager_fused_step_on_host_frames_equal_hbm(strip):
    from test_gpu_23_frame_strips import _sliding_batch
    B, T, N = 8, 80, 24
    H, D = _learners(strip, BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0,
                     LEARNER_DEVICE="cuda:0")
    assert H.memory.store.field_view("state").device.type == "cpu"
    batch = _sliding_batch(N, T, 11)
    for L in (H, D):
        _push(L, batch)
        L.memory.store.seed(5, 0)
    for step in range(2):
        bh, bd = H.memory.sample(), D.memory.sample()
        assert bh[1].is_cuda and torch.equal(bh[1], bd[1])
        info_h, prio_h, idx_h = H.train(bh)
        info_d, prio_d, idx_d = D.train(bd)
        _same(H, D, dict(idx=idx_h, prio=prio_h, scalars=info_h["loss"], p_norm=info_h["p_norm"]),
              dict(idx=idx_d, prio=prio_d, scalars=info_d["loss"], p_norm=info_d["p_norm"]), step)
        H.memory.update(idx_h, prio_h)
        D.memory.update(idx_d, prio_d)
    for step in range(2):
        oh, od = H.fused_step(), D.fused_step()
        torch.cuda.synchronize()
        _same(H, D, oh, od, step)
    assert torch.equal(H.memory.store.priorities(0, N), D.memory.store.priorities(0, N))


@pytest.mark.parametrize("strip", [True, False])
def test_captured_fused_step_on_host_frames_equals_hbm_while_ingest_wraps(strip):
    from test_gpu_23_frame_strips import _sliding_batch
    B, T, N = 8, 80, 32
    H, D = _learners(strip, BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0")
    for L in (H, D):
        _push(L, _sliding_batch(N, T, 21))
        L.memory.store.seed(13, 0)
    for step in range(6):
        if step in (2, 4):                              # ingests that wrap the ring head between replays
            b = _sliding_batch(20, T, 30 + step)
            for L in (H, D):
                _push(L, b)
        oh, od = H.fused_step(use_graph=True), D.fused_step(use_graph=True)
        torch.cuda.synchronize()
        _same(H, D, oh, od, step)
    assert H._graph is not None and D._graph is not None
    assert torch.equal(H.memory.store.priorities(0, N), D.memory.store.priorities(0, N))
    assert torch.equal(H.memory.store.field_view("state"), D.memory.store.field_view("state").cpu())


# ---- served minibatches -----------------------------------------------------------------------------------------------
SLOTS = 6


def test_served_slots_and_served_step_from_host_frames_equal_hbm():
    from fake_redis import FakeRedis
    from test_gpu_19_served_sequences import _bind, _local_memory, _take
    from test_gpu_23_frame_strips import _same_params_and_state, _sliding_batch
    from distributed_rl_b200 import r2d2, replay as R
    from distributed_rl_b200.replay_server import DeviceReplayServer
    B, T, N = 8, 80, 40
    base = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                FRAME_STRIP=True)
    fields = R.r2d2_fields(T, strip=True)
    strips, _, a, r, h0, h1, nd, p = _sliding_batch(N, T, 51)
    servers, learners = [], []
    try:
        for host in (True, False):
            srv = DeviceReplayServer(r2d2.R2D2Config(**base, HOST_FRAMES=host), FakeRedis(), slots=SLOTS)
            servers.append(srv)
            srv._ingest.push_arrays(strips, a, r, h0, h1, nd, p)
            srv.store.seed(7, 0)
            for k in range(SLOTS):
                srv._fill(k, 100 + k)
        torch.cuda.synchronize()
        assert servers[0].store.field_view("state").device.type == "cpu"
        for k in range(SLOTS):
            th, td = _take(servers[0].ring, k, fields, False), _take(servers[1].ring, k, fields, False)
            torch.cuda.synchronize()
            assert torch.equal(th[0], td[0]) and torch.equal(th[1], td[1]) and torch.equal(th[2], td[2]), k
            for f in fields:
                assert torch.equal(th[3][f.name], td[3][f.name]), (k, f.name)
        for srv in servers:
            torch.manual_seed(0)
            learners.append(r2d2.Learner(r2d2.R2D2Config(**base, SERVED_FUSED_STEP=True), start_replay=False,
                                         memory=_local_memory(srv.ring)))
        for k in range(SLOTS):
            outs = []
            for srv, L in zip(servers, learners):
                _bind(srv.ring, k, fields, L._state())
                outs.append(L._bound_step())
            torch.cuda.synchronize()
            for key in ("idx", "prio", "scalars", "p_norm"):
                assert torch.equal(outs[0][key], outs[1][key]), (k, key)
        _same_params_and_state(learners[0].optim, learners[1].optim)
    finally:
        torch.cuda.synchronize()
        for srv in servers:
            srv.close()


# ---- placement and refusals -------------------------------------------------------------------------------------------
def test_placement_footprint_and_refusals():
    from distributed_rl_b200 import _lib, replay as R
    from distributed_rl_b200.replay_server import ServeRing
    lib = _lib.load()
    N, T = 4096, 80
    fields = R.r2d2_fields(T, strip=True)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    st = R.DeviceReplay(N, fields, "cuda:0", host_fields=("state",))
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    small = N * sum(f.nbytes for f in fields if f.name != "state")
    assert small == N * 4_740
    assert used <= small + (64 << 20), used        # small fields + sum-tree + allocation slack, no frames
    for i, f in enumerate(fields):
        flag = ctypes.c_int32(-1)
        _lib.check(lib.b2rl_replay_field_placement(st._h, i, ctypes.byref(flag)))
        assert flag.value == (1 if f.name == "state" else 0)
    view = st.field_view("state")
    assert view.device.type == "cpu" and view.is_pinned()    # is_pinned: cudaPointerGetAttributes says host memory
    assert view.shape == (N, T + 3, 84, 84)
    for name in ("action", "h0"):
        assert st.field_view(name).is_cuda

    frames = R.strip_windows(view)
    pack = R.Conv1Pack(1, "cuda:0")
    launches = lib.b2rl_launch_count()
    with pytest.raises(ValueError, match="host memory"):
        R.conv1_fused(frames, None, pack)
    with pytest.raises(ValueError, match="host memory"):
        R.conv1_wgrad(frames[:4], None, torch.zeros(4, 32, 20, 20, device="cuda"))
    with pytest.raises(_lib.B2RLError, match="host"):
        _lib.check(lib.b2rl_dedup_attach(st._h, 0, 1024, 16, 0))
    st.push(_records(fields, 4, 5)[0], torch.ones(4))   # something to serve
    torch.cuda.synchronize()
    ring = ServeRing.create(st, 4, 2)
    try:
        launches = lib.b2rl_launch_count()
        with pytest.raises(_lib.B2RLError, match="host"):
            ring.fill_uniform(st, 0, 1, T)
        assert lib.b2rl_launch_count() == launches
    finally:
        ring.close()
    # pageable rows are refused by the C entry points before any work (DeviceReplay.push stages them on the device)
    ptrs = (ctypes.c_void_p * _lib.MAX_FIELDS)()
    pageable = np.zeros((1, T + 3, 84, 84), np.uint8)
    ptrs[0] = pageable.ctypes.data
    prio = torch.ones(1, device="cuda")
    head = st.head
    with pytest.raises(_lib.B2RLError, match="pageable"):
        _lib.check(lib.b2rl_replay_push(st._h, ptrs, prio.data_ptr(), 1, torch.cuda.current_stream().cuda_stream))
    with pytest.raises(_lib.B2RLError, match="pageable"):
        _lib.check(lib.b2rl_replay_ingest_pipelined(st._h, ptrs, prio.data_ptr(), 1,
                                                    torch.cuda.current_stream().cuda_stream))
    assert st.head == head and len(st) == 4 and lib.b2rl_launch_count() == launches
    st.close()
