"""GPU tests of the deduplicated R2D2 store with its frame pool in pinned host memory (R.StripDedupReplay(host_pool=True),
R2D2Config.HOST_POOL, DESIGN.md §4.19): the same seeded stream pushed into an HBM-pool store and a host-pool store in
the same chunks gives the same pool ids, head_seq, priorities, live slots and live pool frames, equal to the CPU model
(past the slot ring's wrap and pool-eviction kills, and with every key colliding); gathers equal each other and a
FRAME_STRIP store's; the pool is in host memory; eager and captured fused_step, and served slots with the served
captured step, are bit-identical across the two stores."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from strip_dedup_model import StripDedupModel, player_sequences  # noqa: E402

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


def _stream(n, T, seed, random_tail=0, actors=5):
    strips, a, r, h0, h1, nd, _ = player_sequences(n, T=T, actors=actors, episode=(2 * T, 5 * T), seed=seed)
    rng = np.random.default_rng(seed + 100)
    if random_tail:
        strips[-random_tail:] = rng.integers(0, 256, strips[-random_tail:].shape, dtype=np.uint8)
    p = (rng.random(n) + 0.01).astype(np.float32)
    return strips, a, r, h0, h1, nd, p


def _live_pool_frames(st, live):
    """The pool frames the live slots' plane rows name, in plane order, as a CPU tensor."""
    ids = st.field_view("planes")[torch.from_numpy(live.astype(np.int64)).cuda()].flatten().long().cpu()
    return st.pool[ids] if st.pool.device.type == "cpu" else st.pool[ids.cuda()].cpu()


@pytest.mark.parametrize("mask", [(1 << 63) - 1, 0], ids=["exact", "all_collide"])
def test_host_pool_ids_liveness_and_frames_equal_the_hbm_pool_and_the_model(R, mask):
    T, cap = 16, 64
    Rf = T + 3
    F, W = 40 * Rf, 6 * Rf
    hbm = R.StripDedupReplay(cap, F, W, T=T, hash_mask=mask)
    host = R.StripDedupReplay(cap, F, W, T=T, hash_mask=mask, host_pool=True)
    m = StripDedupModel(cap, F, W, T, mask)
    assert host.max_batch == hbm.max_batch and host.pool.device.type == "cpu" and hbm.pool.is_cuda
    strips, a, r, h0, h1, nd, p = _stream(400, T, seed=11, random_tail=60)
    at = 0
    for b in [13, 1, 40, 7, 33, 25] * 10:
        if at >= len(p):
            break
        sl = slice(at, min(at + b, len(p)))
        for st in (hbm, host):
            x = [torch.from_numpy(v[sl]) for v in (strips, a, r, h0, h1, nd)]
            if b == 7:
                x[0] = x[0].cuda()                            # device strips take the same path
            st.push(x, torch.from_numpy(p[sl]))
        m.push(strips[sl], p[sl])
        at = sl.stop
    torch.cuda.synchronize()
    assert m.head > F and at > 4 * cap                        # both rings wrapped
    for st in (hbm, host):
        assert st.head_seq == m.head and len(st) == m.size and st.head == m.slot_head
        assert torch.equal(st.field_view("planes").cpu(), torch.from_numpy(m.planes))
        assert np.array_equal(st.priorities(0, cap).cpu().numpy(), m.prio)
    live = m.live_slots()
    assert 0 < len(live) < cap                                # the frame rule killed some slots
    frames = _live_pool_frames(host, live)
    assert torch.equal(frames, _live_pool_frames(hbm, live))
    last = {}
    for i in range(at):
        last[i % cap] = i
    rec = np.array([last[int(x)] for x in live])
    assert np.array_equal(frames.numpy().reshape(len(live), Rf, 84, 84), strips[rec])
    idx = torch.from_numpy(live.astype(np.int64)).cuda()
    g0, g1 = hbm.gather(idx), host.gather(idx)
    assert g0.keys() == g1.keys()
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    assert np.array_equal(g1["state"].cpu().numpy(), strips[rec])


def test_gathers_draws_and_priorities_equal_the_strip_store(R):
    T, cap, n = 80, 128, 120
    strips, a, r, h0, h1, nd, p = _stream(n, T, seed=21)
    plain = R.DeviceReplay(cap, R.r2d2_fields(T, strip=True), "cuda:0")
    hbm = R.StripDedupReplay(cap, 80 * cap, 8 * cap, T=T)
    host = R.StripDedupReplay(cap, 80 * cap, 8 * cap, T=T, host_pool=True)
    stores = (plain, hbm, host)
    for st in stores:
        for i in range(0, n, 50):
            st.push([torch.from_numpy(x[i:i + 50]) for x in (strips, a, r, h0, h1, nd)], torch.from_numpy(p[i:i + 50]))
        st.seed(31, 0)
    assert len(plain) == len(hbm) == len(host) == n and hbm.head_seq == host.head_seq
    idx = torch.tensor([0, 119, 5, 5, 64, 1], device="cuda")
    outs = [st.gather(idx) for st in stores]
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]) and torch.equal(outs[0][k], outs[2][k]), k
    for step in range(5):
        draws = [st.sample(32) for st in stores]
        for d in draws[1:]:
            for u, v in zip(draws[0], d):
                assert torch.equal(u, v), step
        new = torch.rand(32, device="cuda") + 0.01
        for st, d in zip(stores, draws):
            st.update(d[0], new)
        g = [st.gather(draws[0][0]) for st in stores]
        assert torch.equal(g[0]["state"], g[2]["state"]) and torch.equal(g[1]["state"], g[2]["state"]), step
    assert torch.equal(plain.priorities(), host.priorities())


def test_the_pool_is_in_host_memory(R):
    from distributed_rl_b200 import _lib
    lib = _lib.load()
    T, cap, F, W = 80, 2048, 150_000, 1024                   # a 1.06 GB pool
    pool_bytes = F * 84 * 84
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    st = R.StripDedupReplay(cap, F, W, T=T, host_pool=True)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    assert used < pool_bytes // 8, used                       # planes, keys, tables, sum-tree: no frames
    flag, ptr = ctypes.c_int32(-1), ctypes.c_void_p()
    _lib.check(lib.b2rl_dedup_pool_placement(st._h, ctypes.byref(flag), ctypes.byref(ptr)))
    assert flag.value == 1 and ptr.value == st.pool.data_ptr()
    assert st.pool.device.type == "cpu" and st.pool.is_pinned()   # is_pinned: cudaPointerGetAttributes says host
    assert st.pool.shape == (F, 84, 84)
    hbm = R.StripDedupReplay(16, 512, 64, T=16)
    _lib.check(lib.b2rl_dedup_pool_placement(hbm._h, ctypes.byref(flag), ctypes.byref(ptr)))
    assert flag.value == 0 and ptr.value == hbm.pool.data_ptr()
    ap = R.DedupReplay(16, 512, 64)
    _lib.check(lib.b2rl_dedup_pool_placement(ap._h, ctypes.byref(flag), None))
    assert flag.value == 0
    # conv_1 never reads a host pool: refused before any launch
    launches = lib.b2rl_launch_count()
    with pytest.raises(ValueError, match="host"):
        st.frame_source("state")
    with pytest.raises(ValueError, match="host memory"):
        R.conv1_fused(R.PlaneFrames(st.pool, st.field_view("planes"), 0, 1), None, R.Conv1Pack(1, "cuda:0"))
    assert lib.b2rl_launch_count() == launches
    # a replay with host fields takes no pool; a handle takes one pool
    hf = R.DeviceReplay(16, R.R2D2_DEDUP_FIELDS(16), "cuda:0", host_fields=("h0",))
    assert lib.b2rl_dedup_attach_strips_placed(hf._h, 0, 19, 512, 64, (1 << 63) - 1, 1) != 0
    assert b"host" in lib.b2rl_last_error()
    assert lib.b2rl_dedup_attach_strips_placed(st._h, 0, T + 3, 512, 64, (1 << 63) - 1, 1) != 0
    assert b"already has a frame pool" in lib.b2rl_last_error()
    st.close()


# ---- the learner ------------------------------------------------------------------------------------------------------
def _learners(**kw):
    """Two learners of the same weights on FRAME_DEDUP stores: pool in HBM, pool in host memory."""
    from distributed_rl_b200 import r2d2
    out = []
    for host in (False, True):
        torch.manual_seed(0)
        out.append(r2d2.Learner(r2d2.R2D2Config(**kw, FRAME_DEDUP=True, HOST_POOL=host), start_replay=False))
    return out


def _same(D, H, od, oh, step):
    from test_gpu_23_frame_strips import _same_params_and_state
    for key in ("idx", "prio", "scalars", "p_norm"):
        assert torch.equal(od[key], oh[key]), (step, key)
    _same_params_and_state(D.optim, H.optim)


def test_eager_and_captured_fused_step_on_a_host_pool_equal_the_hbm_pool(R):
    B, T, N = 8, 80, 32
    kw = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0",
              FRAMES_PER_SEQUENCE=48, DEDUP_WINDOW=192)
    D, H = _learners(**kw)
    assert isinstance(H.memory.store, R.StripDedupReplay) and H.memory.store.host_pool
    assert not D.memory.store.host_pool
    strips, a, r, h0, h1, nd, p = _stream(4 * N, T, seed=41, random_tail=3 * N)
    for L in (D, H):
        L.memory.push_arrays(strips[:N], a[:N], r[:N], h0[:N], h1[:N], nd[:N], p[:N])
        L.memory.store.seed(13, 0)
    for step in range(2):
        od, oh = D.fused_step(), H.fused_step()
        torch.cuda.synchronize()
        _same(D, H, od, oh, step)
    assert D._graph is None and H._graph is None
    at, killed = N, False
    for step in range(7):
        if step in (1, 3, 5):                                # ingest that wraps the ring and kills slots between replays
            sl = slice(at, at + 20)
            for L in (D, H):
                L.memory.push_arrays(strips[sl], a[sl], r[sl], h0[sl], h1[sl], nd[sl], p[sl])
            at += 20
            killed |= len(D.memory.store) < N
        od, oh = D.fused_step(use_graph=True), H.fused_step(use_graph=True)
        torch.cuda.synchronize()
        _same(D, H, od, oh, step)
    assert D._graph is not None and H._graph is not None and killed
    assert len(D.memory.store) == len(H.memory.store)
    assert torch.equal(D.memory.store.priorities(), H.memory.store.priorities())
    for u, v in zip(D.model.parameters(), H.model.parameters()):
        assert torch.equal(u, v)


# ---- served minibatches -----------------------------------------------------------------------------------------------
SLOTS = 6          # 3 eager warm-ups, the capture (replayed once), 2 replays after rebinds


def test_served_slots_from_a_host_pool_and_the_served_step_on_them():
    from fake_redis import FakeRedis
    from test_gpu_19_served_sequences import _bind, _local_memory, _take
    from test_gpu_23_frame_strips import _same_params_and_state
    from distributed_rl_b200 import r2d2, replay as R
    from distributed_rl_b200.replay_server import KINDS, DeviceReplayServer
    B, T, N = 8, 80, 40
    base = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0")
    fields = R.r2d2_fields(T, strip=True)
    strips, a, r, h0, h1, nd, p = _stream(N, T, seed=51)
    servers = []
    try:
        for host in (False, True):
            srv = DeviceReplayServer(r2d2.R2D2Config(**base, FRAME_DEDUP=True, HOST_POOL=host), FakeRedis(),
                                     slots=SLOTS)
            servers.append(srv)
            srv._ingest.push_arrays(strips, a, r, h0, h1, nd, p)
            srv.store.seed(7, 0)
            for k in range(SLOTS):
                srv._fill(k, 100 + k)
        torch.cuda.synchronize()
        assert servers[1].store.pool.device.type == "cpu" and servers[0].store.pool.is_cuda
        assert bytes(servers[0].ring.layout) == bytes(servers[1].ring.layout)
        for k in range(SLOTS):
            bufs = []
            for srv in servers:
                buf = torch.empty(srv.ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
                srv.ring.take(k, buf, torch.cuda.current_stream())
                bufs.append(buf)
            torch.cuda.synchronize()
            assert torch.equal(bufs[0], bufs[1]), k                 # the whole slot, byte for byte
        # the captured bound step on the host pool's slots against train() on a copy of each slot
        ring = servers[1].ring
        torch.manual_seed(0)
        A = r2d2.Learner(r2d2.R2D2Config(**base, FRAME_STRIP=True, SERVED_FUSED_STEP=True), start_replay=False,
                         memory=_local_memory(ring))
        torch.manual_seed(0)
        Bl = r2d2.Learner(r2d2.R2D2Config(**base, FRAME_STRIP=True), start_replay=False)
        s = A._state()
        for k in range(SLOTS):
            _bind(ring, k, fields, s)
            out = A._bound_step()
            hdr, idx, w, b = _take(ring, k, fields, False)
            info, prio, idx_b = Bl.train(KINDS["r2d2"].batch(b, w, idx))
            torch.cuda.synchronize()
            assert hdr.tolist() == [100 + k, B]
            assert torch.equal(out["idx"], idx_b) and torch.equal(out["prio"], prio), k
            assert torch.equal(out["scalars"][0], info["loss"]) and torch.equal(out["p_norm"], info["p_norm"]), k
            _same_params_and_state(A.optim, Bl.optim)
        assert A._graph is not None
    finally:
        torch.cuda.synchronize()
        for srv in servers:
            srv.close()
