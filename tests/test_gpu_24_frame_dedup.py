"""GPU tests of the frame-deduplicated Ape-X store (R.DedupReplay, ApexConfig.FRAME_DEDUP): pool ids against the CPU
model after several wraps of both rings, byte-exact stacks for every live slot, zero priority for dead ones, with
exact and with forced-collision keys; conv_1 over plane tables, and a weight gradient over them split over two
launches; the captured learner step against a stack store."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dedup_model import DedupModel, player_records  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import replay
    return replay


def _stream(n, seed, random_tail=0):
    """Player records; the last `random_tail` have frames that never repeat (they drive the frame-count eviction)."""
    s, ns, a, r, d = player_records(n, actors=9, seed=seed)
    rng = np.random.default_rng(seed + 100)
    if random_tail:
        s[-random_tail:] = rng.integers(0, 256, s[-random_tail:].shape, dtype=np.uint8)
        ns[-random_tail:] = rng.integers(0, 256, ns[-random_tail:].shape, dtype=np.uint8)
    p = rng.random(n).astype(np.float32) + 0.01
    return s, ns, a, r, d, p


@pytest.mark.parametrize("mask", [(1 << 63) - 1, 0], ids=["exact", "all_collide"])
def test_pool_ids_liveness_and_stacks_match_the_model(R, mask):
    cap, F, W = 256, 1024, 128
    st = R.DedupReplay(cap, F, W, hash_mask=mask)
    m = DedupModel(cap, F, W, mask)
    s, ns, a, r, d, p = _stream(1800, seed=11, random_tail=300)
    sizes = [50, 37, 300, 1, 111, 64] * 10
    at = 0
    for b in sizes:
        if at >= len(p):
            break
        sl = slice(at, min(at + b, len(p)))
        host = [torch.from_numpy(x[sl]) for x in (s, ns, a, r, d)]
        if b == 37:
            host[:2] = [t.cuda() for t in host[:2]]          # device stacks take the same path
        st.push(host, torch.from_numpy(p[sl]))
        m.push(s[sl], ns[sl], p[sl])
        at = sl.stop
    torch.cuda.synchronize()
    assert m.head > 2 * F and at > 4 * cap                    # both rings wrapped more than once
    assert st.head_seq == m.head and len(st) == m.size and st.head == m.slot_head
    assert torch.equal(st.field_view("planes").cpu(), torch.from_numpy(m.planes))
    assert np.array_equal(st.priorities(0, cap).cpu().numpy(), m.prio)
    live = m.live_slots()
    assert 0 < len(live) < cap                                 # the frame rule killed some slots
    dead = np.setdiff1d(np.arange(cap), live)
    assert (st.priorities(0, cap).cpu().numpy()[dead] == 0).all()
    idx = torch.from_numpy(live.astype(np.int64)).cuda()
    b = st.gather(idx)
    last = {}
    for i in range(at):
        last[i % cap] = i
    rec = np.array([last[int(x)] for x in live])
    assert np.array_equal(b["state"].cpu().numpy(), s[rec]) and np.array_equal(b["next_state"].cpu().numpy(), ns[rec])
    assert np.array_equal(b["action"].cpu().numpy(), a[rec]) and np.array_equal(b["reward"].cpu().numpy(), r[rec])
    assert np.array_equal(b["done"].cpu().numpy(), d[rec])
    # sampling only ever draws live slots
    st.seed(5, 0)
    drawn, _, _ = st.sample(4096)
    assert np.isin(drawn.cpu().numpy(), live).all()


def test_pipelined_ingest_is_refused(R):
    st = R.DedupReplay(64, 512, 64)
    x = torch.zeros(4, 4, 84, 84, dtype=torch.uint8)
    with pytest.raises(ValueError, match="pipelined"):
        st.ingest_pipelined([x, x, torch.zeros(4, dtype=torch.int32), torch.zeros(4), torch.zeros(4, dtype=torch.uint8)],
                            torch.ones(4))
    with pytest.raises(ValueError, match="pipelined"):
        st.push_begin([x], 4)


@pytest.mark.parametrize("n_nets,c_out,relu", [(1, 32, True), (2, 32, True), (2, 16, False), (1, 16, True)])
def test_conv1_on_plane_tables_equals_rows(R, n_nets, c_out, relu):
    st = R.DedupReplay(512, 2048, 256)
    s, ns, a, r, d = player_records(400, seed=3)
    st.push([torch.from_numpy(x) for x in (s, ns, a, r, d)], torch.ones(400))
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    idx = torch.randint(0, 400, (300,), device="cuda", generator=g)
    idx[:5] = torch.tensor([0, 399, 399, 17, 0])
    batch = st.gather(idx)
    pack = R.Conv1Pack(n_nets, "cuda", c_out)
    for k in range(n_nets):
        pack.pack(k, torch.randn(c_out, 4, 8, 8, device="cuda", generator=g) * 0.05)
    for name in ("state", "next_state"):
        src = st.frame_source(name)
        y_planes = R.conv1_fused(src, idx, pack, relu=relu)
        y_rows = R.conv1_fused(batch[name], None, pack, relu=relu)
        for u, v in zip(y_planes, y_rows):
            assert torch.equal(u, v)
        gy = torch.randn(300, c_out, 20, 20, device="cuda", generator=g)
        ry = y_rows[0] if relu else None
        gw_p = R.conv1_wgrad(src, idx, gy, relu_y=ry)
        gw_r = R.conv1_wgrad(batch[name], None, gy, relu_y=ry)
        assert torch.equal(gw_p, gw_r)
    # all rows in slot order (idx None) against the gathered rows 0..399 of the plane table
    all_rows = torch.arange(512, device="cuda")
    full = st.gather(all_rows)
    y_all = R.conv1_fused(st.frame_source("state"), None, pack, relu=relu)[0]
    assert torch.equal(y_all, R.conv1_fused(full["state"], None, pack, relu=relu)[0])


@pytest.mark.parametrize("accumulate", [False, True])
def test_plane_weight_gradient_split_over_two_launches(R, accumulate):
    """n = SMs * 160 + 257 plane-table rows without idx: the second launch starts 8 * off pool ids into the table."""
    per_launch = torch.cuda.get_device_properties(0).multi_processor_count * 160
    n = per_launch + 257
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    pool = torch.randint(0, 256, (1024, 84, 84), dtype=torch.uint8, device="cuda", generator=g)
    planes = torch.randint(0, 1024, (n, 8), dtype=torch.int32, device="cuda", generator=g)
    src = R.PlaneFrames(pool, planes, 4)
    stacks = pool[planes[:, 4:8].long()]                          # the same rows gathered: (n, 4, 84, 84)
    gy = torch.randn(n, 32, 20, 20, device="cuda", generator=g)
    y = torch.relu(torch.randn(n, 32, 20, 20, device="cuda", generator=g))
    outs = []
    for frames in (stacks, src):
        out = torch.full((32, 4, 8, 8), 0.25, device="cuda")
        outs.append(R.conv1_wgrad(frames, None, gy, out=out, accumulate=accumulate, relu_y=y))
    assert torch.equal(outs[0], outs[1])
    part = R.conv1_wgrad(stacks[:per_launch], None, gy[:per_launch], relu_y=y[:per_launch])
    assert not torch.equal(R.conv1_wgrad(src, None, gy, relu_y=y), part)   # the second launch's rows count
    del stacks, gy, y
    torch.cuda.empty_cache()


def _learner(apex, dedup, B, N):
    cfg = apex.ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                          CUDNN_BENCHMARK=False, FRAME_DEDUP=dedup, DEDUP_WINDOW=1024)
    torch.manual_seed(0)
    L = apex.Learner(cfg, connect=None, start_replay=False)
    with torch.no_grad():
        for p in L.target_model.parameters():
            p.add_(0.01 * torch.randn(p.shape, device=p.device))
    return L


def test_captured_fused_step_is_bit_identical_to_the_stack_store(R):
    from distributed_rl_b200 import apex
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B, N = 64, 2048
    s, ns, a, r, d, p = _stream(3000, seed=21)
    res = []
    for dedup in (False, True):
        L = _learner(apex, dedup, B, N)
        for i in range(0, 3000, 250):
            L.memory.push_arrays(*[torch.from_numpy(x[i:i + 250]) for x in (s, ns, a, r, d, p)])
        st = L.memory.store
        assert isinstance(st, R.DedupReplay) == dedup
        st.seed(77, 0)
        outs = []
        for _ in range(6):
            out = L.fused_step(use_graph=True)
            outs.append({k: v.clone() for k, v in out.items()})
        torch.cuda.synchronize()
        res.append((outs, st.priorities().clone(), [q.detach().clone() for q in L.model.parameters()], len(st)))
    (o0, p0, w0, n0), (o1, p1, w1, n1) = res
    assert n0 == n1 == N
    for a_, b_ in zip(o0, o1):
        for k in a_:
            assert torch.equal(a_[k], b_[k]), k
    assert torch.equal(p0, p1)
    for u, v in zip(w0, w1):
        assert torch.equal(u, v)


def test_push_records_and_buffer_round_trip(R):
    from distributed_rl_b200 import apex
    cfg = apex.ApexConfig(BATCHSIZE=16, REPLAY_MEMORY_LEN=1024, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                          FRAME_DEDUP=True, DEDUP_WINDOW=512)
    rep = apex.Replay(cfg)
    s, ns, a, r, d = player_records(300, seed=5)
    blobs = [pickle.dumps([s[i], int(a[i]), float(r[i]), ns[i], bool(d[i]), 1.0 + i]) for i in range(300)]
    rep.push_records(blobs[:120])
    rep.push_records(blobs[120:])
    torch.cuda.synchronize()
    st = rep.store
    assert len(st) == 300 and st.head_seq < 3 * 300
    idx = torch.arange(300, device="cuda")
    b = st.gather(idx)
    assert np.array_equal(b["state"].cpu().numpy(), s) and np.array_equal(b["next_state"].cpu().numpy(), ns)
    assert np.array_equal(st.priorities(0, 300).cpu().numpy(), 1.0 + np.arange(300, dtype=np.float32))
    rep.buffer(2)
    sb, ab, rb, nsb, db, w, ib = rep.deque[-1]
    k = ib.cpu().numpy()
    assert np.array_equal(sb.cpu().numpy(), s[k]) and np.array_equal(nsb.cpu().numpy(), ns[k])
    with pytest.raises(ValueError, match="pipelined"):
        rep.ingest(*[torch.from_numpy(x[:4]) for x in (s, ns, a, r, d)], torch.ones(4))


def _stores(R, n, cap, seed):
    """A stack store and a dedup store holding the same n Player-like records, the same priorities, seeded alike."""
    s, ns, a, r, d, p = _stream(n, seed=seed)
    stacks = R.DeviceReplay(cap, R.APEX_FIELDS, "cuda:0")
    dedup = R.DedupReplay(cap, 4 * cap, cap // 2)
    for st in (stacks, dedup):
        for i in range(0, n, 100):
            st.push([torch.from_numpy(x[i:i + 100]) for x in (s, ns, a, r, d)], torch.from_numpy(p[i:i + 100]))
        st.seed(31, 0)
    return stacks, dedup


def test_serve_fill_of_a_dedup_store_equals_the_stack_store_slot_for_slot(R):
    """b2rl_serve_fill on a dedup store writes ring slots byte-identical to those of a stack store with the same
    records: the planes field is served as the s and s' stack fields, so the ring layout is APEX_FIELDS'."""
    from distributed_rl_b200.replay_server import ServeRing
    stacks, dedup = _stores(R, 700, 512, seed=41)
    B, slots = 96, 3
    rings = [ServeRing.create(st, B, slots) for st in (stacks, dedup)]
    try:
        L0, L1 = rings[0].layout, rings[1].layout
        assert bytes(L0) == bytes(L1)
        assert [L1.field_bytes[i] for i in range(L1.n_fields)] == [f.nbytes for f in R.APEX_FIELDS]
        for fill in range(7):
            bufs = []
            for st, ring in zip((stacks, dedup), rings):
                ring.fill(st, fill % slots, fill + 1, 0.4)
                buf = torch.empty(ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
                ring.take(fill % slots, buf, torch.cuda.current_stream())
                bufs.append(buf)
            torch.cuda.synchronize()
            assert torch.equal(bufs[0], bufs[1]), fill
        with pytest.raises(R._lib.B2RLError, match="rollouts"):
            rings[1].fill_uniform(dedup, 0, 99, 3)
        with pytest.raises(R._lib.B2RLError, match="b2rl_dedup_push"):
            dedup.build(torch.ones(8, device="cuda"))
    finally:
        torch.cuda.synchronize()
        for ring in rings:
            ring.close()


def test_captured_bound_step_on_dedup_served_slots_is_bit_identical(R):
    """The captured served step (SERVED_FUSED_STEP) bound to ring slots filled from a dedup store and from a stack
    store with the same records: identical bound draws, priorities, scalars and weights after every step."""
    from types import SimpleNamespace
    from distributed_rl_b200 import apex
    from distributed_rl_b200.replay_server import ServeRing
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B, slots, steps = 64, 8, 8
    stores = _stores(R, 900, 1024, seed=43)
    res = []
    for st in stores:
        ring = ServeRing.create(st, B, slots)
        for k in range(slots):
            ring.fill(st, k, k + 1, 0.4)
        torch.manual_seed(0)
        mem = SimpleNamespace(ring=ring, acquire=None, release=None, is_alive=lambda: True)
        L = apex.Learner(apex.ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=8, BUFFER_SIZE=0, CUDNN_BENCHMARK=False,
                                         LEARNER_DEVICE="cuda:0", SERVED_FUSED_STEP=True),
                         start_replay=False, memory=mem)
        s = L._fused_state()
        outs = []
        for k in range(steps):
            ring.bind(ring.slot_ptrs(k % slots)[0][0], R.APEX_FIELDS, s.cur, s.frames, torch.cuda.current_stream())
            out = L.fused_step(use_graph=True)
            outs.append({kk: v.clone() for kk, v in out.items()} | {"w": s.cur["w"].clone()})
        torch.cuda.synchronize()
        assert L._graph is not None
        res.append((outs, [q.detach().clone() for q in L.model.parameters()]))
        ring.close()
    (o0, w0), (o1, w1) = res
    for a_, b_ in zip(o0, o1):
        for k in a_:
            assert torch.equal(a_[k], b_[k]), k
    for u, v in zip(w0, w1):
        assert torch.equal(u, v)
