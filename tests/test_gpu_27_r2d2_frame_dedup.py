"""GPU tests of the frame-deduplicated R2D2 store (R.StripDedupReplay, R2D2Config.FRAME_DEDUP): pool ids, head_seq
and live slots against the CPU model (exact and all-colliding keys, a pool wrap that evicts); gathers, draws and
priorities against a FRAME_STRIP store; conv_1 through a stride-1 plane table against the strip windows; the learner's
eager and captured fused_step against a FRAME_STRIP learner; served slots against a strip store's, and the served
captured step on them; the refusals."""
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


@pytest.mark.parametrize("mask", [(1 << 63) - 1, 0], ids=["exact", "all_collide"])
def test_pool_ids_liveness_and_strips_match_the_model(R, mask):
    T, cap = 16, 64
    Rf = T + 3
    F, W = 40 * Rf, 6 * Rf
    st = R.StripDedupReplay(cap, F, W, T=T, hash_mask=mask)
    m = StripDedupModel(cap, F, W, T, mask)
    assert st.max_batch == min(cap, (F - W - 1) // Rf, 65536 // Rf)
    strips, a, r, h0, h1, nd, p = _stream(400, T, seed=11, random_tail=60)
    at = 0
    for b in [13, 1, 40, 7, 33, 25] * 10:
        if at >= len(p):
            break
        sl = slice(at, min(at + b, len(p)))
        host = [torch.from_numpy(x[sl]) for x in (strips, a, r, h0, h1, nd)]
        if b == 7:
            host[0] = host[0].cuda()                          # device strips take the same path
        st.push(host, torch.from_numpy(p[sl]))
        m.push(strips[sl], p[sl])
        at = sl.stop
    torch.cuda.synchronize()
    assert m.head > F and at > 4 * cap                        # both rings wrapped
    assert st.head_seq == m.head and len(st) == m.size and st.head == m.slot_head
    assert torch.equal(st.field_view("planes").cpu(), torch.from_numpy(m.planes))
    assert np.array_equal(st.priorities(0, cap).cpu().numpy(), m.prio)
    live = m.live_slots()
    assert 0 < len(live) < cap                                # the frame rule killed some slots
    idx = torch.from_numpy(live.astype(np.int64)).cuda()
    b = st.gather(idx)
    last = {}
    for i in range(at):
        last[i % cap] = i
    rec = np.array([last[int(x)] for x in live])
    assert np.array_equal(b["state"].cpu().numpy(), strips[rec])
    for name, x in (("action", a), ("reward", r), ("h0", h0), ("h1", h1), ("notdone", nd)):
        assert np.array_equal(b[name].cpu().numpy(), x[rec]), name
    st.seed(5, 0)
    drawn, _, _ = st.sample(4096)
    assert np.isin(drawn.cpu().numpy(), live).all()


def _stores(R, n, cap, T, seed):
    """A FRAME_STRIP store and a dedup store holding the same n Player-like sequences, seeded alike."""
    strips, a, r, h0, h1, nd, p = _stream(n, T, seed=seed)
    plain = R.DeviceReplay(cap, R.r2d2_fields(T, strip=True), "cuda:0")
    dedup = R.StripDedupReplay(cap, 80 * cap, 8 * cap, T=T)
    for st in (plain, dedup):
        for i in range(0, n, 50):
            st.push([torch.from_numpy(x[i:i + 50]) for x in (strips, a, r, h0, h1, nd)], torch.from_numpy(p[i:i + 50]))
        st.seed(31, 0)
    return plain, dedup


def test_gathers_draws_and_priorities_equal_the_strip_store(R):
    T, cap = 80, 128
    plain, dedup = _stores(R, 120, cap, T, seed=21)
    assert len(plain) == len(dedup) == 120
    strips, *_ = _stream(120, T, seed=21)
    m = StripDedupModel(cap, 80 * cap, 8 * cap, T)
    for i in range(0, 120, 50):
        m.push(strips[i:i + 50], np.ones(min(50, 120 - i), np.float32))
    assert dedup.head_seq == m.head < 0.7 * 120 * (T + 3)         # shared frames are stored once
    idx = torch.tensor([0, 119, 5, 5, 64, 1], device="cuda")
    g0, g1 = plain.gather(idx), dedup.gather(idx)
    assert g0.keys() == g1.keys()
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    for step in range(5):
        (i0, p0, w0), (i1, p1, w1) = plain.sample(32), dedup.sample(32)
        assert torch.equal(i0, i1) and torch.equal(p0, p1) and torch.equal(w0, w1), step
        new = torch.rand(32, device="cuda") + 0.01
        plain.update(i0, new)
        dedup.update(i1, new)
    assert torch.equal(plain.priorities(), dedup.priorities())
    with pytest.raises(ValueError, match="pipelined"):
        dedup.push_begin([None], 4)
    with pytest.raises(ValueError, match="pipelined"):
        dedup.ingest_pipelined(None)
    with pytest.raises(ValueError, match="hashable"):
        dedup.fill_hash(4)
    with pytest.raises(R._lib.B2RLError, match="b2rl_dedup_push"):
        dedup.build(torch.ones(8, device="cuda"))


def test_refusals(R):
    lib = R._lib.load()
    T = 16
    ptrs = (R.C.c_void_p * R._lib.MAX_FIELDS)()
    x = torch.zeros(64, device="cuda")
    ap = R.DedupReplay(16, 512, 64)
    sd = R.StripDedupReplay(16, 512, 64, T=T)
    assert lib.b2rl_dedup_push_strips(ap._h, x.data_ptr(), ptrs, x.data_ptr(), 1, None) != 0
    assert b"b2rl_dedup_push" in lib.b2rl_last_error()
    assert lib.b2rl_dedup_push(sd._h, x.data_ptr(), x.data_ptr(), ptrs, x.data_ptr(), 1, None) != 0
    assert b"b2rl_dedup_push_strips" in lib.b2rl_last_error()
    frames = (R.C.c_void_p * 2)(x.data_ptr(), x.data_ptr())
    idx = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.b2rl_replay_gather_planes(sd._h, idx.data_ptr(), 1, frames, ptrs, None) != 0
    assert b"NULL" in lib.b2rl_last_error()
    fields = R.R2D2_DEDUP_FIELDS(T)
    for bad, msg in ((dict(fpr=T + 2), b"frames_per_record int32"), (dict(pool=T + 3), b"pool_frames - window"),
                     (dict(fpr=2), b"frames_per_record must")):
        h = R.DeviceReplay(16, fields, "cuda:0")
        rc = lib.b2rl_dedup_attach_strips(h._h, 0, bad.get("fpr", T + 3), bad.get("pool", 512), 0, (1 << 63) - 1)
        assert rc != 0 and msg in lib.b2rl_last_error(), msg
    host = R.DeviceReplay(16, R.r2d2_fields(T, strip=True), "cuda:0", host_fields=("state",))
    assert lib.b2rl_dedup_attach_strips(host._h, 0, T + 3, 512, 0, 1) != 0
    with pytest.raises(R._lib.B2RLError, match="rollouts"):
        from distributed_rl_b200.replay_server import ServeRing
        sd.push([torch.zeros(4, T + 3, 84, 84, dtype=torch.uint8), torch.zeros(4, T, dtype=torch.int32),
                 torch.zeros(4, T), torch.zeros(4, 512), torch.zeros(4, 512), torch.ones(4)], torch.ones(4))
        ring = ServeRing.create(sd, 2, 2)
        try:
            ring.fill_uniform(sd, 0, 1, 3)
        finally:
            torch.cuda.synchronize()
            ring.close()
    # plane table descriptors: stride 1 takes base 0 only; other strides are refused
    pool = torch.zeros(16, 84, 84, dtype=torch.uint8, device="cuda")
    planes = torch.zeros(64, dtype=torch.int32, device="cuda")
    pack = R.Conv1Pack(1, "cuda")
    for stride, base, msg in ((1, 4, b"plane_base"), (2, 0, b"plane_stride"), (8, 2, b"plane_base")):
        f = R._lib.Frames(pool=pool.data_ptr(), planes=planes.data_ptr(), plane_base=base, plane_stride=stride, rows=8)
        out = torch.empty(8 * 400 * 32, device="cuda")
        rc = lib.b2rl_conv1_fused(f, None, 8, pack.bq.data_ptr(), pack.scale.data_ptr(), 1, 32, out.data_ptr(), 0,
                                  None)
        assert rc != 0 and msg in lib.b2rl_last_error(), (stride, base)


@pytest.mark.parametrize("n_nets,c_out,relu", [(1, 32, True), (2, 32, False), (2, 16, True)])
def test_conv1_through_a_stride_1_plane_table_equals_strip_windows(R, n_nets, c_out, relu):
    from distributed_rl_b200.learner_common import time_major_rows
    T, cap = 80, 64
    plain, dedup = _stores(R, 64, cap, T, seed=3)
    win = R.strip_windows(plain.field_view("state"))
    src = dedup.frame_source("state")
    assert src.plane_stride == 1 and src.rows == win.shape[0] == cap * (T + 3) - 3
    g = torch.Generator(device="cuda").manual_seed(7)
    pack = R.Conv1Pack(n_nets, "cuda", c_out)
    for k in range(n_nets):
        pack.pack(k, torch.randn(c_out, 4, 8, 8, device="cuda", generator=g) * 0.05)
    seq = torch.tensor([4, 0, 63, 4, 2, 63], device="cuda")
    rows = time_major_rows(seq, torch.arange(T, device="cuda").view(T, 1), T + 3)
    for idx in (rows, torch.tensor([win.shape[0] - 1, 0], device="cuda"), None):
        want = R.conv1_fused(win, idx, pack, relu=relu)
        for u, v in zip(want, R.conv1_fused(src, idx, pack, relu=relu)):
            assert torch.equal(u, v)
        n = win.shape[0] if idx is None else idx.numel()
        gy = torch.randn(n, c_out, 20, 20, device="cuda", generator=g)
        y = want[0] if relu else None
        assert torch.equal(R.conv1_wgrad(win, idx, gy, relu_y=y), R.conv1_wgrad(src, idx, gy, relu_y=y))


@pytest.mark.parametrize("accumulate", [False, True])
def test_weight_gradient_through_a_stride_1_plane_table_split_over_launches(R, accumulate):
    """n = SMs * 160 + 257 windows without idx: the second launch starts off pool ids into the table."""
    per_launch = torch.cuda.get_device_properties(0).multi_processor_count * 160
    n = per_launch + 257
    g = torch.Generator(device="cuda").manual_seed(9)
    pool = torch.randint(0, 256, (2048, 84, 84), dtype=torch.uint8, device="cuda", generator=g)
    planes = torch.randint(0, 2048, (n + 3,), dtype=torch.int32, device="cuda", generator=g)
    src = R.PlaneFrames(pool, planes, 0, 1)
    assert src.rows == n
    stacks = pool[planes.unfold(0, 4, 1).long()]                   # the same windows gathered: (n, 4, 84, 84)
    gy = torch.randn(n, 32, 20, 20, device="cuda", generator=g)
    y = torch.relu(torch.randn(n, 32, 20, 20, device="cuda", generator=g))
    outs = []
    for frames in (stacks, src):
        out = torch.full((32, 4, 8, 8), 0.25, device="cuda")
        outs.append(R.conv1_wgrad(frames, None, gy, out=out, accumulate=accumulate, relu_y=y))
    assert torch.equal(outs[0], outs[1])
    part = R.conv1_wgrad(stacks[:per_launch], None, gy[:per_launch], relu_y=y[:per_launch])
    assert not torch.equal(R.conv1_wgrad(src, None, gy, relu_y=y), part)
    del stacks, gy, y
    torch.cuda.empty_cache()


def _learners(**kw):
    from distributed_rl_b200 import r2d2
    out = []
    for dedup in (False, True):
        torch.manual_seed(0)
        out.append(r2d2.Learner(r2d2.R2D2Config(**kw, FRAME_STRIP=True, FRAME_DEDUP=dedup, FRAMES_PER_SEQUENCE=120,
                                                DEDUP_WINDOW=1024), start_replay=False))
    return out


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "captured"])
def test_fused_step_equals_the_strip_learner(R, use_graph):
    B, T, N = 16, 80, 96
    S, D = _learners(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0")
    assert isinstance(D.memory.store, R.StripDedupReplay) and not isinstance(S.memory.store, R.StripDedupReplay)
    strips, a, r, h0, h1, nd, p = _stream(N + 30, T, seed=41)
    stacks = R.strip_stacks(torch.from_numpy(strips)).contiguous().numpy()
    for L in (S, D):
        L.memory.push_arrays(strips[:50], a[:50], r[:50], h0[:50], h1[:50], nd[:50], p[:50])
        L.memory.push_arrays(stacks[50:], a[50:], r[50:], h0[50:], h1[50:], nd[50:], p[50:])   # stacks encoded
        L.memory.store.seed(13, 0)
    assert len(D.memory.store) == N                             # every slot live
    for step in range(5):
        o0, o1 = S.fused_step(use_graph=use_graph), D.fused_step(use_graph=use_graph)
        torch.cuda.synchronize()
        for key in ("idx", "prio", "scalars", "p_norm"):
            assert torch.equal(o0[key], o1[key]), (step, key)
    assert (S._graph is not None) == (D._graph is not None) == use_graph
    assert torch.equal(S.memory.store.priorities(), D.memory.store.priorities())
    for u, v in zip(S.model.parameters(), D.model.parameters()):
        assert torch.equal(u, v)
    # train() through Replay.buffer: the gathered strips, as a strip store's
    for L in (S, D):
        L.memory.store.seed(3, 0)
        L.memory.buffer(1)
    bs, bd = S.memory.deque.pop(), D.memory.deque.pop()
    assert torch.equal(bs[1], bd[1]) and torch.equal(bs[-1], bd[-1])
    (_, p0, i0), (_, p1, i1) = S.train(bs), D.train(bd)
    assert torch.equal(p0, p1) and torch.equal(i0, i1)


def test_served_slots_equal_the_strip_store_and_the_served_step_runs(R):
    from test_gpu_19_served_sequences import _bind, _local_memory
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200.replay_server import ServeRing
    T, B, slots = 80, 8, 4
    plain, dedup = _stores(R, 90, 128, T, seed=51)
    rings = [ServeRing.create(st, B, slots) for st in (plain, dedup)]
    try:
        assert bytes(rings[0].layout) == bytes(rings[1].layout)
        assert rings[1].layout.field_bytes[0] == (T + 3) * 7056
        for fill in range(2 * slots):
            bufs = []
            for st, ring in zip((plain, dedup), rings):
                ring.fill(st, fill % slots, fill + 1, 0.4)
                buf = torch.empty(ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
                ring.take(fill % slots, buf, torch.cuda.current_stream())
                bufs.append(buf)
            torch.cuda.synchronize()
            assert torch.equal(bufs[0], bufs[1]), fill
        # the captured served step (SERVED_FUSED_STEP) on slots filled from each store: the same bits
        fields = R.r2d2_fields(T, strip=True)
        res = []
        for st, ring in zip((plain, dedup), rings):
            st.seed(7, 0)
            for k in range(slots):
                ring.fill(st, k, 100 + k, 0.4)
            torch.manual_seed(0)
            L = r2d2.Learner(r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=8,
                                             LEARNER_DEVICE="cuda:0", FRAME_STRIP=True, SERVED_FUSED_STEP=True),
                             start_replay=False, memory=_local_memory(ring))
            s = L._state()
            outs = []
            for k in range(2 * slots):
                _bind(ring, k % slots, fields, s)
                out = L._bound_step()
                outs.append({kk: v.clone() for kk, v in out.items()})
            torch.cuda.synchronize()
            assert L._graph is not None
            res.append((outs, [q.detach().clone() for q in L.model.parameters()]))
        (o0, w0), (o1, w1) = res
        for a_, b_ in zip(o0, o1):
            for k in a_:
                assert torch.equal(a_[k], b_[k]), k
        for u, v in zip(w0, w1):
            assert torch.equal(u, v)
    finally:
        torch.cuda.synchronize()
        for ring in rings:
            ring.close()
