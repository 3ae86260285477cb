"""GPU tests of the coded IMPALA frame pool (R.RolloutDedupReplay(pool_bytes=...), ImpalaConfig.STAGED_POOL_CODEC,
DESIGN.md §4.23), against a raw RolloutDedupReplay fed the same rollouts and against the CPU models (the unit-ring strip
model at R = 4 (T + 1), impala_atari_rollouts.staging_map): pool ids, liveness, uniform draws and gathers; the staged
pool (b2rl_dedup_stage_rollouts) and conv_1's forward and weight gradient through it; staging every slot, live, dead or
never written, and a ring of random bytes; the eager and captured learner steps at B = 32 and B = 1024; served slots,
the served step on them and a DeviceReplayServer built with STAGED_POOL_CODEC."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pool_codec_model as M                                   # noqa: E402
from impala_atari_rollouts import atari_rollouts, staging_map  # noqa: E402
from impala_rollouts import rollout_frames                     # noqa: E402

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


def _stream(n, T, seed, random_tail=0):
    """n Player-like rollouts of synthetic Atari-like frames (padded episode ends included), the last `random_tail`
    of random frames (stored raw), as host arrays: state, action, mu, reward, done."""
    state, a, mu, r, done, kind = atari_rollouts(n, T=T, actors=6, episode=(2 * T, 6 * T), p_done=0.3 / T, seed=seed)
    assert "padded" in kind
    if random_tail:
        rng = np.random.default_rng(seed + 100)
        state[-random_tail:] = rng.integers(0, 256, state[-random_tail:].shape, dtype=np.uint8)
    return [state, a, mu, r, done]


def _push(stores, cols, chunks):
    n, at = len(cols[-1]), 0
    for b in chunks:
        if at >= n:
            break
        sl = slice(at, min(at + b, n))
        for st in stores:
            st.push([torch.from_numpy(x[sl]) for x in cols], torch.ones(sl.stop - sl.start))
        at = sl.stop
    return at


def _buffers(B, T):
    from test_gpu_29_impala_frame_dedup import _buffers as buffers
    return buffers(B, T)


def _pair(R, cap, T, F, W, cols, chunks=(50,) * 100):
    """A raw and a coded rollout store of the default ring, (F + 1) x 7 072 bytes, holding the same rollouts."""
    raw = R.RolloutDedupReplay(cap, F, W, T=T)
    coded = R.RolloutDedupReplay(cap, F, W, T=T, pool_bytes=(F + 1) * 7072)
    at = _push((raw, coded), cols, chunks)
    for st in (raw, coded):
        st.seed(31, 0)
    torch.cuda.synchronize()
    return raw, coded, at


def test_ids_liveness_draws_and_gathers_equal_the_raw_store(R):
    T, cap, B = 20, 128, 32
    Rf = 4 * (T + 1)
    F, W = 24 * cap, 512
    cols = _stream(400, T, seed=21, random_tail=20)
    raw, coded, at = _pair(R, cap, T, F, W, cols, [13, 1, 40, 7, 33, 25] * 20)
    assert coded.coded and not raw.coded and coded.pool.dim() == 1 and coded.pool.numel() == (F + 1) * 7072
    assert coded.max_batch == raw.max_batch
    assert raw.head_seq > F and at > 2 * cap                           # both rings wrapped
    assert coded.head_seq == raw.head_seq and len(coded) == len(raw) and coded.head == raw.head
    assert 0 < len(raw) < cap                                          # the frame rule killed slots
    assert torch.equal(coded.field_view("planes"), raw.field_view("planes"))
    assert torch.equal(coded.priorities(), raw.priorities())
    live = torch.nonzero(raw.priorities(0, cap) > 0).flatten()
    g0, g1 = raw.gather(live), coded.gather(live)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    rec = np.arange(at - len(live), at)
    order = np.argsort((live.cpu().numpy() - raw.head + len(live)) % cap)
    assert np.array_equal(g1["state"].cpu().numpy()[order].reshape(len(live), -1), cols[0][rec].reshape(len(live), -1))
    for call in range(3):
        o0, o1 = _buffers(B, T), _buffers(B, T)
        raw.uniform_fetch(B, T, o0)
        coded.uniform_fetch(B, T, o1)
        torch.cuda.synchronize()
        for k in o0:
            assert torch.equal(o0[k], o1[k]), (call, k)
    s = coded.codec_stats()
    assert s["frames_stored"] == coded.head_seq and 16 <= s["bytes_per_frame"] <= 7072
    with pytest.raises(ValueError, match="encoded"):
        coded.frame_source("state")
    with pytest.raises(ValueError, match="coded frame pool"):
        raw.stage_frames(live, {})
    assert Rf == coded.alloc_staged(2)["planes"].shape[1]
    raw.close()
    coded.close()


def test_a_small_coded_pool_equals_the_unit_ring_model(R):
    T, cap, F, W = 4, 96, 4000, 32
    Rf = 4 * (T + 1)
    P = (W + 2 + 3 * Rf) * 442 + 37 * 16                              # the byte rule binds; not a multiple of a frame
    coded = R.RolloutDedupReplay(cap, F, W, T=T, pool_bytes=16 * P)
    m = M.CodedStripDedupModel(cap, F, W, 4 * T + 1, P)
    assert coded.max_batch == M.coded_max_batch(cap, F, W, Rf, P) == 3
    cols = _stream(300, T, seed=17)
    cols[0][::2, 1] = np.random.default_rng(1).integers(0, 256, cols[0][::2, 1].shape, dtype=np.uint8)   # raw frames
    at = 0
    for b in [3, 1, 2, 3, 3] * 100:
        if at >= 300:
            break
        sl = slice(at, min(at + b, 300))
        coded.push([torch.from_numpy(x[sl]) for x in cols], torch.ones(sl.stop - sl.start))
        m.push(rollout_frames(cols[0][sl]), np.ones(sl.stop - sl.start, np.float32))
        at = sl.stop
    torch.cuda.synchronize()
    s = coded.codec_stats()
    assert s["units_written"] == m.units > P and s["pool_units"] == P
    assert coded.head_seq == m.head and len(coded) == m.size and coded.head == m.slot_head
    assert torch.equal(coded.field_view("planes").cpu(), torch.from_numpy(m.planes))
    live = m.live_slots()
    assert 0 < len(live) < min(cap, at)                                 # the byte rule killed slots
    idx = torch.from_numpy(live.astype(np.int64)).cuda()
    g = coded.gather(idx)
    assert np.array_equal(g["state"].cpu().numpy().reshape(len(live), Rf, 84, 84), m.strips(live))
    staged = coded.alloc_staged(len(live))
    src = coded.stage_frames(idx, staged)
    torch.cuda.synchronize()
    want = staging_map(m.planes[live], F)
    assert np.array_equal(staged["planes"].cpu().numpy(), want)
    pool = staged["pool"].cpu().numpy()
    stacks = pool[want.reshape(-1)].reshape(len(live), Rf, 84, 84)      # read through the staged plane table
    assert np.array_equal(stacks, m.strips(live))
    assert src.plane_stride == 4 and src.base == 0 and src.rows == len(live) * (T + 1)
    coded.close()


@pytest.mark.parametrize("n_nets,c_out", [(1, 16), (2, 32)])
def test_conv1_through_the_staged_pool_equals_the_raw_store(R, n_nets, c_out):
    from distributed_rl_b200.learner_common import time_major_rows
    T, cap, B = 20, 64, 24
    cols = _stream(64, T, seed=3)
    raw, coded, _ = _pair(R, cap, T, 40 * cap, 1024, cols)
    out = _buffers(B, T)
    coded.uniform_fetch(B, T, out)
    staged = coded.alloc_staged(B)
    src = coded.stage_frames(out["idx"], staged)
    t_idx = torch.arange(T + 1, device="cuda").view(T + 1, 1)
    rows = time_major_rows(torch.arange(B, device="cuda"), t_idx)
    raw_src, raw_rows = raw.frame_source("state"), out["rows"]
    assert torch.equal(raw_rows, time_major_rows(out["idx"], t_idx))
    distinct = torch.unique(staged["planes"]).numel()
    assert distinct < B * (T + 8)                                       # about T + 1 of 4 (T + 1) frames decoded
    g = torch.Generator(device="cuda").manual_seed(7)
    pack = R.Conv1Pack(n_nets, "cuda", c_out)
    for k in range(n_nets):
        pack.pack(k, torch.randn(c_out, 4, 8, 8, device="cuda", generator=g) * 0.05)
    for relu in (False, True):
        want = R.conv1_fused(raw_src, raw_rows, pack, relu=relu)
        got = R.conv1_fused(src, rows, pack, relu=relu)
        for u, v in zip(want, got):
            assert torch.equal(u, v), relu
        gy = torch.randn(rows.numel(), c_out, 20, 20, device="cuda", generator=g)
        y = want[0] if relu else None
        assert torch.equal(R.conv1_wgrad(raw_src, raw_rows, gy, relu_y=y), R.conv1_wgrad(src, rows, gy, relu_y=y))
        seq = rows[:T * B]                                              # the grad pass's rows, as the learner's
        gy2 = gy[:T * B].contiguous()
        assert torch.equal(R.conv1_wgrad(raw_src, raw_rows[:T * B], gy2, relu_y=None),
                           R.conv1_wgrad(src, seq, gy2, relu_y=None))
    raw.close()
    coded.close()


def test_staging_every_slot_and_random_bytes_stays_inside_the_pool(R):
    """stage_frames takes any slot: never written (zeros), killed by the byte rule (ids naming entries whose offsets
    now fall inside newer encodings), or out of range (clamped).  It completes and the live slots keep their rollouts;
    then a ring of random bytes and random ids in the plane table stage without a fault."""
    T, cap, F, W = 4, 96, 4000, 32
    Rf = 4 * (T + 1)
    P = (W + 2 + 3 * Rf) * 442 + 37 * 16
    coded = R.RolloutDedupReplay(cap, F, W, T=T, pool_bytes=16 * P)
    every = torch.arange(cap, device="cuda")
    staged = coded.alloc_staged(cap)
    coded.stage_frames(every, staged)
    torch.cuda.synchronize()
    read = staged["pool"][staged["planes"].view(-1).long()]             # what conv_1 reads through the staged table
    assert not read.any()                                               # every id 0, decoded from zeroed bytes
    assert torch.equal(staged["planes"], (every.view(-1, 1) * Rf).to(torch.int32).expand(cap, Rf))
    cols = _stream(200, T, seed=23)
    cols[0][::2, 2] = np.random.default_rng(2).integers(0, 256, cols[0][::2, 2].shape, dtype=np.uint8)
    at = _push((coded,), cols, [3] * 100)
    torch.cuda.synchronize()
    n = len(coded)
    assert 0 < n < min(cap, at) and coded.codec_stats()["units_written"] > P
    live = (coded.head - n + np.arange(n)) % cap
    src = coded.stage_frames(every, staged)
    torch.cuda.synchronize()
    planes = staged["planes"].cpu().numpy()
    stacks = staged["pool"].cpu().numpy()[planes.reshape(-1)].reshape(cap, T + 1, 28224)
    assert np.array_equal(stacks[live], cols[0][at - n:at])
    out = coded.alloc_staged(4)
    coded.stage_frames(torch.tensor([-5, cap + 7, 0, cap - 1], device="cuda"), out)
    torch.cuda.synchronize()
    sp = out["planes"].cpu().numpy() - (np.arange(4) * Rf)[:, None]
    assert np.array_equal(sp[0], planes[0]) and np.array_equal(sp[2], planes[0])       # clamped to slot 0
    assert np.array_equal(sp[1], planes[cap - 1] - (cap - 1) * Rf) and np.array_equal(sp[3], sp[1])
    gen = torch.Generator("cuda").manual_seed(9)
    coded.pool.copy_(torch.randint(0, 256, coded.pool.shape, dtype=torch.uint8, device="cuda", generator=gen))
    coded.field_view("planes").copy_(torch.randint(-2 ** 31, 2 ** 31 - 1, coded.field_view("planes").shape,
                                                   dtype=torch.int32, device="cuda", generator=gen))
    coded.stage_frames(every, staged)
    torch.cuda.synchronize()
    want = staging_map(coded.field_view("planes").cpu().numpy(), F)
    assert np.array_equal(staged["planes"].cpu().numpy(), want)
    assert src.rows == cap * (T + 1)
    coded.close()


def test_stage_is_one_launch_and_captures(R):
    T, cap, B = 20, 64, 16
    cols = _stream(64, T, seed=5)
    raw, coded, _ = _pair(R, cap, T, 40 * cap, 1024, cols)
    lib = R._lib.load()
    idx = torch.zeros(B, dtype=torch.int64, device="cuda")
    staged = coded.alloc_staged(B)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        n0 = lib.b2rl_launch_count()
        with torch.cuda.graph(graph, stream=s):
            coded.stage_frames(idx, staged)
        assert lib.b2rl_launch_count() == n0 + 1
    torch.cuda.current_stream().wait_stream(s)
    for k in range(3):
        sel = torch.randperm(cap, device="cuda")[:B]
        idx.copy_(sel)
        graph.replay()
        torch.cuda.synchronize()
        stacks = staged["pool"][staged["planes"].view(-1).long()].reshape(B, -1)
        assert torch.equal(stacks, raw.gather(sel)["state"].reshape(B, -1)), k
    raw.close()
    coded.close()


def _learners(**kw):
    """Two learners of the same weights on FRAME_DEDUP stores: raw pool, coded pool."""
    from distributed_rl_b200 import impala
    out = []
    for codec in (False, True):
        torch.manual_seed(0)
        out.append(impala.Learner(impala.ImpalaConfig(**kw, FRAME_DEDUP=True, STAGED_POOL_CODEC=codec),
                                  start_replay=False))
    return out


@pytest.mark.parametrize("B,N,fpr,tail", [(32, 96, 24.0, 12), (1024, 1100, 40.0, 0)], ids=["B32", "B1024"])
def test_eager_and_captured_steps_equal_the_raw_store(R, B, N, fpr, tail):
    from test_gpu_19_served_sequences import _same_params_and_state
    T = 20
    D, H = _learners(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0",
                     FRAMES_PER_ROLLOUT=fpr, DEDUP_WINDOW=256)
    assert H.memory.store.coded and not D.memory.store.coded
    cols = _stream(N + 3 * 40, T, seed=41, random_tail=tail)
    for L in (D, H):
        L.memory.push_arrays(*[x[:N] for x in cols])
        L.memory.store.seed(13, 0)
    for step in range(2):
        o0, o1 = D.fused_step(), H.fused_step()
        torch.cuda.synchronize()
        for key in ("vtarget", "advantage", "objActor", "criticLoss"):
            assert torch.equal(o0[key], o1[key]), (step, key)
    at, killed = N, False
    for step in range(7):
        if step in (1, 3, 5):                   # ingest that wraps the slot ring (and with random frames the pools)
            sl = slice(at, at + 40)
            for L in (D, H):
                L.memory.push_arrays(*[x[sl] for x in cols])
            at += 40
            killed |= len(D.memory.store) < N
        o0, o1 = D.fused_step(use_graph=True), H.fused_step(use_graph=True)
        torch.cuda.synchronize()
        for key in ("vtarget", "advantage", "objActor", "criticLoss", "idx"):
            assert torch.equal(o0[key], o1[key]), (step, key)
    assert D._graph is not None and H._graph is not None and killed == bool(tail)
    assert len(D.memory.store) == len(H.memory.store) and D.memory.store.head == H.memory.store.head
    if tail:                                    # the frame pool wrapped
        assert H.memory.store.head_seq > H.memory.store.pool_frames
    _same_params_and_state(D.mOptim, H.mOptim)
    assert H._staged.buffers["pool"].shape == (B * 4 * (T + 1), 84, 84)


def test_served_slots_the_served_step_and_a_server_on_a_coded_pool(R):
    from test_gpu_19_served_sequences import _bind, _local_memory, _same_params_and_state
    from test_gpu_17_impala_serve import _impala_record
    from fake_redis import FakeRedis
    from distributed_rl_b200 import impala
    from distributed_rl_b200.replay_server import DeviceReplayServer, ServeRing
    T, slots = 20, 6
    cols = _stream(240, T, seed=61)
    raw, coded, _ = _pair(R, 256, T, 40 * 256, 1024, cols)
    for B in (8, 200):                          # below and above the SM count: the fill's item and draw splits
        rings = [ServeRing.create(st, B, 3) for st in (raw, coded)]
        try:
            assert bytes(rings[0].layout) == bytes(rings[1].layout)
            for fill in range(6):
                bufs = []
                for st, ring in zip((raw, coded), rings):
                    ring.fill_uniform(st, fill % 3, fill + 1, T)
                    buf = torch.empty(ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
                    ring.take(fill % 3, buf, torch.cuda.current_stream())
                    bufs.append(buf)
                torch.cuda.synchronize()
                assert torch.equal(bufs[0], bufs[1]), (B, fill)
            with pytest.raises(R._lib.B2RLError, match="steps"):
                rings[1].fill_uniform(coded, 0, 99, T - 1)
        finally:
            torch.cuda.synchronize()
            for ring in rings:
                ring.close()
    # the served captured step on slots filled from the coded store equals the one on the raw store's
    B = 16
    rings = [ServeRing.create(st, B, slots) for st in (raw, coded)]
    fields = R.impala_fields(T)
    try:
        res = []
        for st, ring in zip((raw, coded), rings):
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
    raw.close()
    coded.close()
    # a DeviceReplayServer built with STAGED_POOL_CODEC ingests the actors' records into the coded store and serves them
    conn = FakeRedis()
    cfg = impala.ImpalaConfig(BATCHSIZE=4, UNROLL_STEP=T, REPLAY_MEMORY_LEN=32, BUFFER_SIZE=8, LEARNER_DEVICE="cuda:0",
                              FRAME_DEDUP=True, STAGED_POOL_CODEC=True, FRAMES_PER_ROLLOUT=100, DEDUP_WINDOW=64)
    srv = DeviceReplayServer(cfg, conn, slots=2)
    try:
        assert isinstance(srv.store, R.RolloutDedupReplay) and srv.store.coded
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


def test_refusals_on_a_device(R):
    lib = R._lib.load()
    T = 4
    ro = R.RolloutDedupReplay(16, 512, 64, T=T)
    co = R.RolloutDedupReplay(16, 512, 64, T=T, pool_bytes=513 * 7072)
    sd = R.StripDedupReplay(16, 512, 64, T=16, pool_bytes=513 * 7072)
    idx = torch.zeros(2, dtype=torch.int64, device="cuda")
    pool = torch.zeros(2 * 20 * 7056 + 16, dtype=torch.uint8, device="cuda")
    planes = torch.zeros(2 * 20 + 1, dtype=torch.int32, device="cuda")
    n0 = lib.b2rl_launch_count()
    for st in (ro, sd):                                                # a raw rollout store, a coded strip store
        assert lib.b2rl_dedup_stage_rollouts(st._h, idx.data_ptr(), 2, pool.data_ptr(), planes.data_ptr(), None) != 0
        assert b"not a coded rollout frame pool" in lib.b2rl_last_error()
    for args, msg in (((None, pool.data_ptr(), planes.data_ptr()), b"null argument"),
                      ((idx.data_ptr(), pool.data_ptr() + 8, planes.data_ptr()), b"16-byte aligned"),
                      ((idx.data_ptr(), pool.data_ptr(), planes.data_ptr() + 2), b"4-byte aligned")):
        assert lib.b2rl_dedup_stage_rollouts(co._h, args[0], 2, args[1], args[2], None) != 0
        assert msg in lib.b2rl_last_error(), msg
    assert lib.b2rl_dedup_stage_rollouts(co._h, idx.data_ptr(), 1 << 27, pool.data_ptr(), planes.data_ptr(), None) != 0
    assert b"2^31" in lib.b2rl_last_error()
    assert lib.b2rl_dedup_stage_rollouts(co._h, idx.data_ptr(), 0, pool.data_ptr(), planes.data_ptr(), None) == 0
    assert lib.b2rl_launch_count() == n0
    with pytest.raises(ValueError, match="alloc_staged"):
        co.stage_frames(idx, {"pool": pool, "planes": planes})
    # the coded rollout attach refuses a handle that already has a pool, as the raw one does
    for st in (ro, co):
        assert lib.b2rl_dedup_attach_rollouts_coded(st._h, 0, T + 1, 512, 64, 1, 513 * 7072) != 0
        assert b"already has a frame pool" in lib.b2rl_last_error()
    with pytest.raises(R._lib.B2RLError, match="b2rl_dedup_push"):
        co.build(torch.ones(8, device="cuda"))
    torch.cuda.synchronize()
