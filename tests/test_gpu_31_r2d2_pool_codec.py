"""GPU tests of the deduplicated R2D2 store with its frames stored encoded (R.StripDedupReplay(pool_bytes=...),
R2D2Config.POOL_CODEC, DESIGN.md §4.21): b2rl_frame_encode writes the numpy encoder's bytes and b2rl_frame_decode
inverts it; with a pool large enough that only the frame rule binds, a coded store equals a plain FRAME_DEDUP store on
the same stream (ids, head_seq, len, gathers, draws, priorities); with a small pool its live slots and strips equal the
unit-ring model's past the wrap; eager and captured fused_step equal the plain store's; served slots are byte for byte
the plain store's and the served captured step runs on them."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pool_codec_model as M                                           # noqa: E402

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


def _stream(n, T, seed, random_tail=0, actors=4):
    """Synthetic Atari-like sequences (compressible), the last `random_tail` replaced by random frames (raw)."""
    strips, a, r, h0, h1, nd, _ = M.atari_sequences(n, T=T, actors=actors, episode=(2 * T, 4 * T), seed=seed)
    rng = np.random.default_rng(seed + 100)
    if random_tail:
        strips[-random_tail:] = rng.integers(0, 256, strips[-random_tail:].shape, dtype=np.uint8)
    p = (rng.random(n) + 0.01).astype(np.float32)
    return strips, a, r, h0, h1, nd, p


def _codec_inputs():
    rng = np.random.default_rng(3)
    frames = [rng.integers(0, 256, (84, 84), dtype=np.uint8) for _ in range(3)]
    frames += [np.full((84, 84), v, np.uint8) for v in (0, 77, 255)]
    for r, x in ((0, 0), (0, 83), (83, 0), (83, 83), (40, 41)):
        f = np.full((84, 84), 7, np.uint8)
        f[r, x] = 200
        frames.append(f)
    alt = np.zeros((84, 84), np.uint8)
    alt[:, ::2] = 255
    chk = alt.copy()
    chk[1::2] = 255 - chk[1::2]
    frames += [alt, chk, np.repeat(np.arange(84, dtype=np.uint8)[:, None] // 21, 84, axis=1)]
    frames += [M.atari_frame(k, ep) for ep in (0, 5) for k in (0, 1, 63, 250)]
    return np.stack(frames)


def test_encode_kernel_writes_the_numpy_encoding_and_decode_inverts_it(R):
    frames = _codec_inputs()
    enc, units = R.encode_frames(torch.from_numpy(frames).cuda())
    torch.cuda.synchronize()
    enc, units = enc.cpu().numpy(), units.cpu().numpy()
    for j, f in enumerate(frames):
        e = M.encode(f)
        assert units[j] == len(e) // 16, j
        assert np.array_equal(enc[j, :len(e)], e), j
    ref = np.zeros((len(frames), M.RAW_BYTES), np.uint8)
    for j, f in enumerate(frames):
        e = M.encode(f)
        ref[j, :len(e)] = e
    out = R.decode_frames(torch.from_numpy(ref).cuda()).cpu().numpy()
    assert np.array_equal(out, frames)
    assert units[:3].tolist() == [442] * 3 and units[3:6].tolist() == [2] * 3


def _push_all(stores, strips, a, r, h0, h1, nd, p, chunks):
    at = 0
    for b in chunks:
        if at >= len(p):
            break
        sl = slice(at, min(at + b, len(p)))
        for st in stores:
            x = [torch.from_numpy(v[sl]) for v in (strips, a, r, h0, h1, nd)]
            st.push(x, torch.from_numpy(p[sl]))
        at = sl.stop
    return at


def test_a_large_coded_pool_equals_the_plain_dedup_store(R):
    T, cap = 16, 64
    Rf = T + 3
    F, W = 40 * Rf, 6 * Rf
    plain = R.StripDedupReplay(cap, F, W, T=T)
    coded = R.StripDedupReplay(cap, F, W, T=T, pool_bytes=(F + 1) * 7072)
    assert coded.max_batch == plain.max_batch and coded.pool.dim() == 1 and coded.pool.numel() == (F + 1) * 7072
    strips, a, r, h0, h1, nd, p = _stream(400, T, seed=11, random_tail=60)
    at = _push_all((plain, coded), strips, a, r, h0, h1, nd, p, [13, 1, 40, 7, 33, 25] * 12)
    torch.cuda.synchronize()
    assert plain.head_seq > F and at > 4 * cap                 # both rings wrapped
    assert coded.head_seq == plain.head_seq and len(coded) == len(plain) and coded.head == plain.head
    assert torch.equal(coded.field_view("planes"), plain.field_view("planes"))
    assert torch.equal(coded.priorities(), plain.priorities())
    assert 0 < len(plain) < cap                                # the frame rule killed some slots
    live = torch.nonzero(plain.priorities(0, cap) > 0).flatten()
    g0, g1 = plain.gather(live), coded.gather(live)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    for st in (plain, coded):
        st.seed(31, 0)
    for step in range(4):
        d0, d1 = plain.sample(32), coded.sample(32)
        for u, v in zip(d0, d1):
            assert torch.equal(u, v), step
        new = torch.rand(32, device="cuda") + 0.01
        plain.update(d0[0], new)
        coded.update(d1[0], new)
        assert torch.equal(plain.gather(d0[0])["state"], coded.gather(d1[0])["state"]), step
    s = coded.codec_stats()
    assert s["frames_stored"] == coded.head_seq and 16 <= s["bytes_per_frame"] <= 7072
    with pytest.raises(ValueError, match="encoded"):
        coded.frame_source("state")
    coded.close()
    plain.close()


def test_a_small_coded_pool_equals_the_unit_ring_model(R):
    T, cap, F, W = 16, 96, 4000, 32
    Rf = T + 3
    P = (W + 2 + 3 * Rf) * 442 + 37 * 16                       # the byte rule binds; not a multiple of a frame
    coded = R.StripDedupReplay(cap, F, W, T=T, pool_bytes=16 * P)
    m = M.CodedStripDedupModel(cap, F, W, T, P)
    assert coded.max_batch == M.coded_max_batch(cap, F, W, Rf, P) == 3
    strips, a, r, h0, h1, nd, p = _stream(200, T, seed=17)
    strips[::11, 4] = np.random.default_rng(1).integers(0, 256, strips[::11, 4].shape, dtype=np.uint8)
    at = 0
    for b in [3, 1, 2, 3, 3] * 60:
        if at >= len(p):
            break
        sl = slice(at, min(at + b, len(p)))
        coded.push([torch.from_numpy(v[sl]) for v in (strips, a, r, h0, h1, nd)], torch.from_numpy(p[sl]))
        m.push(strips[sl], p[sl])
        at = sl.stop
    torch.cuda.synchronize()
    s = coded.codec_stats()
    assert s["units_written"] == m.units > P and s["pool_units"] == P
    assert coded.head_seq == m.head and len(coded) == m.size and coded.head == m.slot_head
    assert torch.equal(coded.field_view("planes").cpu(), torch.from_numpy(m.planes))
    assert np.array_equal(coded.priorities(0, cap).cpu().numpy(), m.prio)
    live = m.live_slots()
    assert 0 < len(live) < min(cap, at)                         # the byte rule killed slots
    g = coded.gather(torch.from_numpy(live.astype(np.int64)).cuda())
    assert np.array_equal(g["state"].cpu().numpy(), m.strips(live))
    assert np.array_equal(g["state"].cpu().numpy(), strips[at - len(live):at])
    ring = coded.pool.cpu().numpy()                             # the ring's bytes are the model's where frames live
    for e in np.unique(m.planes[live]):
        a0, n = 16 * (int(m.foff[e]) % P), 16 * int(m.flen[e])
        assert np.array_equal(ring[a0:a0 + n], m.ring[a0:a0 + n]), e
    coded.close()


def test_every_slot_decodes_inside_the_pool_live_or_dead(R):
    """gather() takes any slot: one never written, or one the byte rule killed, whose ids name entries whose offsets
    now fall inside newer encodings.  Such a gather completes and the live slots keep their sequences; an unwritten
    slot decodes to zeros; and arbitrary bytes decode (row-run kind with row 0's repeat bit set, other kinds)."""
    T, cap, F, W = 16, 96, 4000, 32
    Rf = T + 3
    P = (W + 2 + 3 * Rf) * 442 + 37 * 16
    coded = R.StripDedupReplay(cap, F, W, T=T, pool_bytes=16 * P)
    every = torch.arange(cap, device="cuda")
    g = coded.gather(every)
    torch.cuda.synchronize()
    assert not g["state"].any()
    strips, a, r, h0, h1, nd, p = _stream(150, T, seed=23)
    strips[::7, 2] = np.random.default_rng(2).integers(0, 256, strips[::7, 2].shape, dtype=np.uint8)   # raw frames
    at = _push_all((coded,), strips, a, r, h0, h1, nd, p, [3] * 50)
    torch.cuda.synchronize()
    n = len(coded)
    assert 0 < n < min(cap, at) and coded.codec_stats()["units_written"] > P   # wrapped; the byte rule killed slots
    live = (coded.head - n + np.arange(n)) % cap
    g = coded.gather(every)
    g_out = coded.gather(torch.tensor([-5, cap + 7, 0, cap - 1], device="cuda"))     # clamped into the slot range
    torch.cuda.synchronize()
    assert np.array_equal(g["state"].cpu().numpy()[live], strips[at - n:at])
    assert torch.equal(g_out["state"][0], g["state"][0]) and torch.equal(g_out["state"][1], g["state"][cap - 1])
    enc = torch.randint(0, 256, (256, 7072), dtype=torch.uint8, device="cuda",
                        generator=torch.Generator("cuda").manual_seed(9))
    enc[:192, 0] = 1                                            # row-run headers over random masks and literals
    enc[:96, 3] |= 1                                            # with row 0 marked as a repeat
    enc[192:, 0] = torch.arange(2, 66, dtype=torch.uint8, device="cuda")   # kinds 2..65
    out = R.decode_frames(enc)
    torch.cuda.synchronize()
    assert out.shape == (256, 84, 84)
    assert torch.equal(out[192:], enc[192:, 16:].reshape(64, 84, 84))   # any other kind reads as raw
    coded.close()


# ---- the learner ------------------------------------------------------------------------------------------------------
def _learners(**kw):
    """Two learners of the same weights on FRAME_DEDUP stores: raw pool, coded pool."""
    from distributed_rl_b200 import r2d2
    out = []
    for codec in (False, True):
        torch.manual_seed(0)
        out.append(r2d2.Learner(r2d2.R2D2Config(**kw, FRAME_DEDUP=True, POOL_CODEC=codec), start_replay=False))
    return out


def _same(D, H, od, oh, step):
    from test_gpu_23_frame_strips import _same_params_and_state
    for key in ("idx", "prio", "scalars", "p_norm"):
        assert torch.equal(od[key], oh[key]), (step, key)
    _same_params_and_state(D.optim, H.optim)


def test_eager_and_captured_fused_step_on_a_coded_pool_equal_the_plain_pool(R):
    B, T, N = 8, 80, 32
    kw = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0",
              FRAMES_PER_SEQUENCE=48, DEDUP_WINDOW=192)
    D, H = _learners(**kw)
    assert H.memory.store.coded and not D.memory.store.coded
    strips, a, r, h0, h1, nd, p = _stream(4 * N, T, seed=41, random_tail=N)
    for L in (D, H):
        L.memory.push_arrays(strips[:N], a[:N], r[:N], h0[:N], h1[:N], nd[:N], p[:N])
        L.memory.store.seed(13, 0)
    for step in range(2):
        od, oh = D.fused_step(), H.fused_step()
        torch.cuda.synchronize()
        _same(D, H, od, oh, step)
    at, killed = N, False
    for step in range(7):
        if step in (1, 3, 5):                                # ingest that wraps the ring and kills slots between replays
            sl = slice(at, at + 30)
            for L in (D, H):
                L.memory.push_arrays(strips[sl], a[sl], r[sl], h0[sl], h1[sl], nd[sl], p[sl])
            at += 30
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


def test_served_slots_from_a_coded_pool_and_the_served_step_on_them():
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
        for codec in (False, True):
            srv = DeviceReplayServer(r2d2.R2D2Config(**base, FRAME_DEDUP=True, POOL_CODEC=codec), FakeRedis(),
                                     slots=SLOTS)
            servers.append(srv)
            srv._ingest.push_arrays(strips, a, r, h0, h1, nd, p)
            srv.store.seed(7, 0)
            for k in range(SLOTS):
                srv._fill(k, 100 + k)
        torch.cuda.synchronize()
        assert servers[1].store.coded and not servers[0].store.coded
        assert bytes(servers[0].ring.layout) == bytes(servers[1].ring.layout)
        for k in range(SLOTS):
            bufs = []
            for srv in servers:
                buf = torch.empty(srv.ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
                srv.ring.take(k, buf, torch.cuda.current_stream())
                bufs.append(buf)
            torch.cuda.synchronize()
            assert torch.equal(bufs[0], bufs[1]), k                 # the whole slot, byte for byte
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
