"""GPU tests of the frame-deduplicated IMPALA store (R.RolloutDedupReplay, ImpalaConfig.FRAME_DEDUP, DESIGN.md §4.20):
pool ids, head_seq, live slots and gathered rows against the CPU model (tests/impala_rollouts.py: the strip model at
R = 4 (T + 1); exact and all-colliding keys, pushes above max_batch, a pool wrap that kills slots, draws from live
slots only); gathers and
uniform draws against a stack store's and against tests/uniform_oracle.py; conv_1 and its weight gradient through the
stride-4 plane table against the stack store's rows; served slots against a stack store's, and a DeviceReplayServer
built from the config; the learner's eager and captured fused_step, train() and the served captured step against a
stack-store learner; the refusals."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from impala_rollouts import player_rollouts, rollout_frames, rollout_model  # noqa: E402
from uniform_oracle import uniform_draw  # noqa: E402

pytestmark = pytest.mark.gpu

SMALL = ("action", "mu", "reward", "done")


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


def _stream(n, T, seed, random_tail=0):
    """n Player-like rollouts (padded episode ends included) as host arrays: state, action, mu, reward, done."""
    state, a, mu, r, done, kind = player_rollouts(n, T=T, actors=6, episode=(2 * T, 6 * T), p_done=0.3 / T, seed=seed)
    assert "padded" in kind
    if random_tail:
        rng = np.random.default_rng(seed + 100)
        state[-random_tail:] = rng.integers(0, 256, state[-random_tail:].shape, dtype=np.uint8)
    return [state, a, mu, r, done]


def _push(st, cols, chunk=50):
    n = len(cols[-1])
    for i in range(0, n, chunk):
        st.push([torch.from_numpy(x[i:i + chunk]) for x in cols], torch.ones(min(chunk, n - i)))


def _stores(R, n, cap, T, seed):
    """A stack store and a dedup store holding the same n Player-like rollouts, their Philox streams seeded alike."""
    cols = _stream(n, T, seed)
    plain = R.DeviceReplay(cap, R.impala_fields(T), "cuda:0")
    dedup = R.RolloutDedupReplay(cap, 40 * cap, 1024, T=T)       # F - W above the pushes' frames: no slot dies
    for st in (plain, dedup):
        _push(st, cols)
        st.seed(31, 0)
    torch.cuda.synchronize()
    return plain, dedup, cols


def _buffers(B, T):
    from distributed_rl_b200.replay import impala_fields
    f = {x.name: x for x in impala_fields(T)}
    out = {name: torch.zeros((T, B), dtype=f[name].dtype, device="cuda") for name in ("action", "mu", "reward")}
    out.update(done=torch.zeros(B, dtype=f["done"].dtype, device="cuda"),
               idx=torch.zeros(B, dtype=torch.int64, device="cuda"),
               rows=torch.zeros((T + 1) * B, dtype=torch.int64, device="cuda"))
    return out


@pytest.mark.parametrize("mask", [(1 << 63) - 1, 0], ids=["exact", "all_collide"])
def test_pool_ids_liveness_and_rows_match_the_model(R, mask):
    T, cap = 4, 64
    Rf = 4 * (T + 1)
    F, W = 40 * Rf, 6 * Rf
    st = R.RolloutDedupReplay(cap, F, W, T=T, hash_mask=mask)
    m = rollout_model(cap, F, W, T, mask)
    assert st.max_batch == min(cap, (F - W - 1) // Rf, 65536 // Rf) == 33
    cols = _stream(400, T, seed=11, random_tail=60)
    at = 0
    for b in [13, 1, 40, 7, 33, 25] * 10:                     # 40 > max_batch: pushed in two chunks
        if at >= 400:
            break
        sl = slice(at, min(at + b, 400))
        host = [torch.from_numpy(x[sl]) for x in cols]
        if b == 7:
            host[0] = host[0].cuda()                          # device rows take the same path
        st.push(host, torch.ones(sl.stop - sl.start))
        m.push(rollout_frames(cols[0][sl]), np.ones(sl.stop - sl.start, np.float32))
        at = sl.stop
    torch.cuda.synchronize()
    assert m.head > F and at > 4 * cap                        # both rings wrapped
    assert st.head_seq == m.head and len(st) == m.size and st.head == m.slot_head
    assert torch.equal(st.field_view("planes").cpu(), torch.from_numpy(m.planes))
    assert torch.equal(st.pool.cpu(), torch.from_numpy(m.pool))
    live = m.live_slots()
    assert 0 < len(live) < cap                                # the frame rule killed some slots
    idx = torch.from_numpy(live.astype(np.int64)).cuda()
    b = st.gather(idx)
    rec = np.arange(at - len(live), at)                       # the live slots hold the newest rollouts
    for name, x in zip(("state",) + SMALL, cols):
        assert np.array_equal(b[name].cpu().numpy(), x[rec]), name
    # draws without replacement see the live slots only: a draw of every live slot is a permutation of them
    out = _buffers(len(live), T)
    for seed in (5, 6):
        st.seed(seed, 0)
        st.uniform_fetch(len(live), T, out)
        assert sorted(out["idx"].tolist()) == sorted(live.tolist())
    with pytest.raises(ValueError, match="larger than population"):
        st.uniform_fetch(len(live) + 1, T, _buffers(len(live) + 1, T))


def test_gathers_and_uniform_draws_equal_the_stack_store(R):
    T, cap, B = 20, 128, 32
    plain, dedup, cols = _stores(R, 120, cap, T, seed=21)
    assert len(plain) == len(dedup) == 120
    assert dedup.head_seq < 0.3 * 120 * 4 * (T + 1)                 # shared frames are stored once
    idx = torch.tensor([0, 119, 5, 5, 64, 1], device="cuda")
    g0, g1 = plain.gather(idx), dedup.gather(idx)
    assert g0.keys() == g1.keys()
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    size, _, head = dedup._sizes()
    for call in range(3):
        o0, o1 = _buffers(B, T), _buffers(B, T)
        plain.uniform_fetch(B, T, o0)
        dedup.uniform_fetch(B, T, o1)
        torch.cuda.synchronize()
        for k in o0:
            assert torch.equal(o0[k], o1[k]), (call, k)
        np.testing.assert_array_equal(o1["idx"].cpu().numpy(), uniform_draw(31, call * B, B, size, cap, head))
    src = dedup.frame_source("state")
    assert src.plane_stride == 4 and src.rows == cap * (T + 1)


@pytest.mark.parametrize("n_nets,c_out", [(1, 16), (2, 32)])
def test_conv1_through_a_stride_4_plane_table_equals_the_stack_rows(R, n_nets, c_out):
    from distributed_rl_b200.learner_common import time_major_rows
    T, cap = 20, 64
    plain, dedup, _ = _stores(R, 64, cap, T, seed=3)
    stacks = plain.field_view("state").view(-1, 4, 84, 84)
    src = dedup.frame_source("state")
    g = torch.Generator(device="cuda").manual_seed(7)
    pack = R.Conv1Pack(n_nets, "cuda", c_out)
    for k in range(n_nets):
        pack.pack(k, torch.randn(c_out, 4, 8, 8, device="cuda", generator=g) * 0.05)
    seq = torch.tensor([4, 0, 63, 4, 2, 63], device="cuda")
    rows = time_major_rows(seq, torch.arange(T + 1, device="cuda").view(T + 1, 1))
    for idx in (rows, torch.tensor([cap * (T + 1) - 1, 0], device="cuda"), None):
        for relu in (False, True):
            want = R.conv1_fused(stacks, idx, pack, relu=relu)
            for u, v in zip(want, R.conv1_fused(src, idx, pack, relu=relu)):
                assert torch.equal(u, v), relu
            n = stacks.shape[0] if idx is None else idx.numel()
            gy = torch.randn(n, c_out, 20, 20, device="cuda", generator=g)
            y = want[0] if relu else None
            assert torch.equal(R.conv1_wgrad(stacks, idx, gy, relu_y=y), R.conv1_wgrad(src, idx, gy, relu_y=y))


@pytest.mark.parametrize("B", [8, 200])
def test_served_slots_equal_the_stack_store(R, B):
    """b2rl_serve_fill_uniform from a dedup store: the same slot bytes as from a stack store (B below and above the SM
    count: the item split and the draw split of the fill)."""
    from distributed_rl_b200.replay_server import ServeRing
    T, slots = 20, 3
    plain, dedup, _ = _stores(R, 240, 256, T, seed=51)
    rings = [ServeRing.create(st, B, slots) for st in (plain, dedup)]
    try:
        assert bytes(rings[0].layout) == bytes(rings[1].layout)
        assert rings[1].layout.field_bytes[0] == (T + 1) * 28224
        for fill in range(2 * slots):
            bufs = []
            for st, ring in zip((plain, dedup), rings):
                ring.fill_uniform(st, fill % slots, fill + 1, T)
                buf = torch.empty(ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
                ring.take(fill % slots, buf, torch.cuda.current_stream())
                bufs.append(buf)
            torch.cuda.synchronize()
            assert torch.equal(bufs[0], bufs[1]), fill
        with pytest.raises(R._lib.B2RLError, match="steps"):
            rings[1].fill_uniform(dedup, 0, 99, T - 1)
    finally:
        torch.cuda.synchronize()
        for ring in rings:
            ring.close()


def _learners(**kw):
    from distributed_rl_b200 import impala
    out = []
    for dedup in (False, True):
        torch.manual_seed(0)
        out.append(impala.Learner(impala.ImpalaConfig(**kw, FRAME_DEDUP=dedup, FRAMES_PER_ROLLOUT=40,
                                                      DEDUP_WINDOW=256), start_replay=False))
    return out


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "captured"])
def test_fused_step_equals_the_stack_learner(R, use_graph):
    from test_gpu_19_served_sequences import _same_params_and_state
    B, T, N = 16, 20, 96
    S, D = _learners(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0")
    assert isinstance(D.memory.store, R.RolloutDedupReplay) and not isinstance(S.memory.store, R.RolloutDedupReplay)
    cols = _stream(N + 30, T, seed=41)
    for L in (S, D):
        L.memory.push_arrays(*[x[:50] for x in cols])
        L.memory.push_arrays(*[torch.from_numpy(x[50:]).pin_memory() for x in cols])   # wraps the slot ring
        L.memory.store.seed(13, 0)
    assert len(D.memory) == len(S.memory) == N                  # every slot live
    for step in range(5):
        o0, o1 = S.fused_step(use_graph=use_graph), D.fused_step(use_graph=use_graph)
        torch.cuda.synchronize()
        for key in ("vtarget", "advantage", "objActor", "criticLoss") + (("idx",) if use_graph else ()):
            assert torch.equal(o0[key], o1[key]), (step, key)
    assert (S._graph is not None) == (D._graph is not None) == use_graph
    _same_params_and_state(S.mOptim, D.mOptim)
    # train() through Replay.bufferSave: the gathered rollouts, as a stack store's
    for L in (S, D):
        L.memory.bufferSave(1)
    bs, bd = S.memory.deque.pop(), D.memory.deque.pop()
    for u, v in zip(bs, bd):
        assert torch.equal(u, v)
    S.train(bs)
    D.train(bd)
    torch.cuda.synchronize()
    for key in ("vtarget", "advantage", "objActor", "criticLoss"):
        assert torch.equal(S.last[key], D.last[key]), key
    _same_params_and_state(S.mOptim, D.mOptim)


def test_served_captured_step_equals_the_stack_store_and_a_server_serves_rollouts(R):
    from test_gpu_19_served_sequences import _bind, _local_memory, _same_params_and_state
    from test_gpu_17_impala_serve import _impala_record
    from fake_redis import FakeRedis
    from distributed_rl_b200 import impala
    from distributed_rl_b200.replay_server import DeviceReplayServer, ServeRing
    T, B, slots = 20, 16, 6
    plain, dedup, _ = _stores(R, 90, 128, T, seed=61)
    rings = [ServeRing.create(st, B, slots) for st in (plain, dedup)]
    fields = R.impala_fields(T)
    try:
        res = []
        for st, ring in zip((plain, dedup), rings):
            st.seed(7, 0)
            for k in range(slots):
                ring.fill_uniform(st, k, 100 + k, T)
            torch.manual_seed(0)
            L = impala.Learner(impala.ImpalaConfig(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=8,
                                                   LEARNER_DEVICE="cuda:0", SERVED_FUSED_STEP=True),
                               start_replay=False, memory=_local_memory(ring))
            s = L._bound_state()
            outs = []
            for k in range(slots):
                _bind(ring, k, fields, s)
                outs.append({kk: v.clone() for kk, v in L._bound_step().items()})
            torch.cuda.synchronize()
            assert L._graph is not None
            res.append((outs, L))
        (o0, L0), (o1, L1) = res
        for a_, b_ in zip(o0, o1):
            for k in ("vtarget", "advantage", "objActor", "criticLoss"):
                assert torch.equal(a_[k], b_[k]), k
        _same_params_and_state(L0.mOptim, L1.mOptim)
    finally:
        torch.cuda.synchronize()
        for ring in rings:
            ring.close()
    # a DeviceReplayServer built with FRAME_DEDUP ingests the actors' records into the dedup store and serves them
    conn = FakeRedis()
    cfg = impala.ImpalaConfig(BATCHSIZE=4, UNROLL_STEP=T, REPLAY_MEMORY_LEN=32, BUFFER_SIZE=8, LEARNER_DEVICE="cuda:0",
                              FRAME_DEDUP=True, FRAMES_PER_ROLLOUT=100, DEDUP_WINDOW=64)
    srv = DeviceReplayServer(cfg, conn, slots=2)
    try:
        assert isinstance(srv.store, R.RolloutDedupReplay)
        rng = np.random.default_rng(0)
        recs = [_impala_record(rng, T) for _ in range(12)]
        conn.rpush("trajectory", *[pickle.dumps(r) for r in recs])
        st = srv.serve_once()
        assert st["ingested"] == 12 and st["filled"] >= 1 and len(srv.store) == 12
        buf = torch.empty(srv.ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
        srv.ring.take(0, buf, torch.cuda.current_stream())
        torch.cuda.synchronize()
        L = srv.ring.layout
        idx = buf[L.idx_off:L.idx_off + 32].view(torch.int64)
        state = buf[L.field_off[0]:L.field_off[0] + 4 * (T + 1) * 28224].view(T + 1, 4, 28224)
        want = np.stack([recs[i][0] for i in idx.tolist()], axis=1)          # (T + 1, B, 28224) time-major
        assert np.array_equal(state.cpu().numpy(), want)
    finally:
        torch.cuda.synchronize()
        srv.close(timeout=0)


def test_refusals(R):
    from distributed_rl_b200.replay_server import ServeRing
    lib = R._lib.load()
    T = 4
    ptrs = (R.C.c_void_p * R._lib.MAX_FIELDS)()
    x = torch.zeros(64, device="cuda")
    ro = R.RolloutDedupReplay(16, 512, 64, T=T)
    cols = _stream(12, T, seed=1)
    _push(ro, cols)
    # the other dedup stores still serve no rollouts, and hold none to fetch
    ap = R.DedupReplay(16, 512, 64)
    ap.push([torch.zeros(4, 4, 84, 84, dtype=torch.uint8)] * 2 + [torch.zeros(4, dtype=torch.int32), torch.zeros(4),
                                                                   torch.zeros(4, dtype=torch.uint8)], torch.ones(4))
    sd = R.StripDedupReplay(16, 512, 64, T=16)
    sd.push([torch.zeros(4, 19, 84, 84, dtype=torch.uint8), torch.zeros(4, 16, dtype=torch.int32), torch.zeros(4, 16),
             torch.zeros(4, 512), torch.zeros(4, 512), torch.ones(4)], torch.ones(4))
    idx = torch.zeros(2, dtype=torch.int64, device="cuda")
    for st, steps in ((ap, 3), (sd, 16)):
        ring = ServeRing.create(st, 2, 1)
        try:
            with pytest.raises(R._lib.B2RLError, match="prioritized minibatches, not rollouts"):
                ring.fill_uniform(st, 0, 1, steps)
        finally:
            torch.cuda.synchronize()
            ring.close()
        assert lib.b2rl_uniform_fetch(st._h, 2, steps, idx.data_ptr(), None, None, None) != 0
        assert b"holds no rollouts" in lib.b2rl_last_error()
    assert lib.b2rl_uniform_fetch(ro._h, 2, T + 1, idx.data_ptr(), None, None, None) != 0
    assert b"steps + 1" in lib.b2rl_last_error()
    planes_out = (R.C.c_void_p * R._lib.MAX_FIELDS)(x.data_ptr())
    assert lib.b2rl_uniform_fetch(ro._h, 2, T, idx.data_ptr(), planes_out, None, None) != 0
    assert b"read in place" in lib.b2rl_last_error()
    # the rollout store's own refusals: the Ape-X push, tree build, pipelined ingest, payload hashing, host fields
    assert lib.b2rl_dedup_push(ro._h, x.data_ptr(), x.data_ptr(), ptrs, x.data_ptr(), 1, None) != 0
    assert b"b2rl_dedup_push_strips" in lib.b2rl_last_error()
    with pytest.raises(R._lib.B2RLError, match="b2rl_dedup_push"):
        ro.build(torch.ones(8, device="cuda"))
    with pytest.raises(ValueError, match="pipelined"):
        ro.push_begin([None], 4)
    with pytest.raises(ValueError, match="pipelined"):
        ro.ingest_pipelined(None)
    with pytest.raises(ValueError, match="hashable"):
        ro.fill_hash(4)
    fields = R.IMPALA_DEDUP_FIELDS(T)
    for stacks, msg in ((T, b"frames_per_record int32"), (0, b"stacks_per_record"), (20000, b"stacks_per_record")):
        h = R.DeviceReplay(16, fields, "cuda:0")
        rc = lib.b2rl_dedup_attach_rollouts(h._h, 0, stacks, 512, 0, (1 << 63) - 1)
        assert rc != 0 and msg in lib.b2rl_last_error(), msg
    host = R.DeviceReplay(16, R.impala_fields(T), "cuda:0", host_fields=("state",))
    assert lib.b2rl_dedup_attach_rollouts(host._h, 0, T + 1, 512, 0, 1) != 0
    assert b"host" in lib.b2rl_last_error()
    # plane table descriptors: stride 4 takes base 0 only; strides other than 1, 4 and 8 are refused
    pool = torch.zeros(16, 84, 84, dtype=torch.uint8, device="cuda")
    planes = torch.zeros(64, dtype=torch.int32, device="cuda")
    pack = R.Conv1Pack(1, "cuda", 16)
    for stride, base, msg in ((4, 4, b"plane_base"), (2, 0, b"plane_stride"), (3, 0, b"plane_stride")):
        f = R._lib.Frames(pool=pool.data_ptr(), planes=planes.data_ptr(), plane_base=base, plane_stride=stride, rows=8)
        out = torch.empty(8 * 400 * 16, device="cuda")
        rc = lib.b2rl_conv1_fused(f, None, 8, pack.bq.data_ptr(), pack.scale.data_ptr(), 1, 16, out.data_ptr(), 0,
                                  None)
        assert rc != 0 and msg in lib.b2rl_last_error(), (stride, base)
    torch.cuda.synchronize()
