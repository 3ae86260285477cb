"""GPU tests of the coded Ape-X frame pool (R.CodedDedupReplay, ApexConfig.FRAME_CODEC, DESIGN.md §4.22): the store
against the unit-ring model and a raw DedupReplay (ids, liveness, priorities, gathered s / s'), with a large ring and
with the byte rule binding past several wraps; conv_1's forward and weight gradient on the coded frame source bit for
bit against the raw source and, on dead and never-written slots, against conv_1 on the gathered stacks; random pool
bytes; the eager and captured learner steps and the served fill and bound step against a raw dedup store."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from apex_atari_records import atari_records              # noqa: E402
from pool_codec_model import CodedStripDedupModel          # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import replay
    return replay


def _stream(n, seed):
    s, ns, a, r, d = atari_records(n, actors=9, seed=seed)
    p = np.random.default_rng(seed + 100).random(n).astype(np.float32) + 0.01
    return s, ns, a, r, d, p


def _push_both(stores, model, recs, sizes):
    s, ns, a, r, d, p = recs
    at = 0
    for b in sizes:
        if at >= len(p):
            break
        sl = slice(at, min(at + b, len(p)))
        for st in stores:
            st.push([torch.from_numpy(x[sl]) for x in (s, ns, a, r, d)], torch.from_numpy(p[sl]))
        if model is not None:
            model.push(np.concatenate([s[sl], ns[sl]], axis=1), p[sl])
        at = sl.stop
    torch.cuda.synchronize()
    return at


@pytest.mark.parametrize("ring", ["large", "binding"])
def test_store_matches_the_model_and_the_raw_store(R, ring):
    if ring == "large":                                      # the frame and slot rules bind, never the byte rule
        cap, F, W = 256, 1024, 64
        P = (F + 1) * 442
    else:                                                    # a ring of (W + 2 + 32) raw frames binds
        cap, F, W = 1024, 1024, 16
        P = (W + 2 + 8 * 4) * 442
    coded = R.CodedDedupReplay(cap, F, W, 16 * P)
    raw = R.DedupReplay(cap, F, W)
    m = CodedStripDedupModel(cap, F, W, 5, P)                 # T = 5: R = 8 frames per record
    recs = _stream(3000, seed=11)
    at = _push_both((coded, raw), m, recs, [50, 37, 120, 1, 64] * 20)
    st = coded.codec_stats()
    assert st["frames_stored"] == m.head == coded.head_seq and st["units_written"] == m.units
    assert m.head > 2 * F
    if ring == "binding":
        assert m.units > 3 * P                               # several wraps of the unit ring
    assert torch.equal(coded.field_view("planes").cpu(), torch.from_numpy(m.planes.reshape(cap, 8)))
    assert np.array_equal(coded.priorities(0, cap).cpu().numpy(), m.prio)
    live = m.live_slots()
    if ring == "large":                                      # the byte rule never binds: the raw store's slots
        assert torch.equal(coded.field_view("planes"), raw.field_view("planes"))
        assert torch.equal(coded.priorities(0, cap), raw.priorities(0, cap))
    else:
        assert len(live) < len(raw)
    idx = torch.from_numpy(live.astype(np.int64)).cuda()
    b = coded.gather(idx)
    both = m.strips(live)
    s, ns = both[:, :4], both[:, 4:]
    assert np.array_equal(b["state"].cpu().numpy(), s) and np.array_equal(b["next_state"].cpu().numpy(), ns)
    last = {}
    for i in range(at):
        last[i % cap] = i
    rec = np.array([last[int(x)] for x in live])
    assert np.array_equal(b["state"].cpu().numpy(), recs[0][rec])
    assert np.array_equal(b["next_state"].cpu().numpy(), recs[1][rec])
    assert np.array_equal(b["action"].cpu().numpy(), recs[2][rec])


def _packs(R, n_nets, c_out, g):
    pack = R.Conv1Pack(n_nets, "cuda", c_out)
    for k in range(n_nets):
        pack.pack(k, torch.randn(c_out, 4, 8, 8, device="cuda", generator=g) * 0.05)
    return pack


@pytest.mark.parametrize("n", [512, 301])
@pytest.mark.parametrize("n_nets,c_out,relu", [(1, 32, True), (2, 32, False), (2, 16, True), (1, 16, False)])
def test_conv1_on_the_coded_source_equals_the_raw_source(R, n, n_nets, c_out, relu):
    cap, F, W = 1024, 4096, 256
    coded, raw = R.CodedDedupReplay(cap, F, W, 16 * (W + 2 + 8 * 40) * 442), R.DedupReplay(cap, F, W)
    _push_both((coded, raw), None, _stream(700, seed=3), [100] * 7)
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    idx = torch.randint(0, 700, (n,), device="cuda", generator=g)
    idx[:4] = torch.tensor([0, 699, 699, 17])
    pack = _packs(R, n_nets, c_out, g)
    for name in ("state", "next_state"):
        yc = R.conv1_fused(coded.frame_source(name), idx, pack, relu=relu)
        yr = R.conv1_fused(raw.frame_source(name), idx, pack, relu=relu)
        for u, v in zip(yc, yr):
            assert torch.equal(u, v), name
        gy = torch.randn(n, c_out, 20, 20, device="cuda", generator=g)
        ry = yr[0] if relu else None
        assert torch.equal(R.conv1_wgrad(coded.frame_source(name), idx, gy, relu_y=ry),
                           R.conv1_wgrad(raw.frame_source(name), idx, gy, relu_y=ry))
    # dead and never-written slots (700..1023, and the clamped -5 / 5000) decode the bytes gather decodes
    idx2 = torch.cat([torch.arange(650, 1024, device="cuda"), torch.tensor([-5, 5000], device="cuda")])
    b = coded.gather(idx2)
    for name in ("state", "next_state"):
        yc = R.conv1_fused(coded.frame_source(name), idx2, pack, relu=relu)
        yg = R.conv1_fused(b[name], None, pack, relu=relu)
        for u, v in zip(yc, yg):
            assert torch.equal(u, v), name


@pytest.mark.parametrize("accumulate", [False, True])
def test_coded_weight_gradient_split_over_two_launches(R, accumulate):
    per_launch = torch.cuda.get_device_properties(0).multi_processor_count * 160
    n = per_launch + 257                                       # rows 0..n-1 without idx: two launches
    cap, F, W = n, 8 * 1024, 512
    coded, raw = R.CodedDedupReplay(cap, F, W, 16 * (W + 2 + 8 * 64) * 442 * 4), R.DedupReplay(cap, F, W)
    _push_both((coded, raw), None, _stream(3000, seed=5), [500] * 6)
    g = torch.Generator(device="cuda"); g.manual_seed(9)
    gy = torch.randn(n, 32, 20, 20, device="cuda", generator=g)
    y = torch.relu(torch.randn(n, 32, 20, 20, device="cuda", generator=g))
    for ry in (None, y):
        outs = []
        for st in (coded, raw):
            out = torch.full((32, 4, 8, 8), 0.25, device="cuda")
            outs.append(R.conv1_wgrad(st.frame_source("next_state"), None, gy, out=out, accumulate=accumulate,
                                      relu_y=ry))
        assert torch.equal(outs[0], outs[1])


def test_random_pool_bytes_decode_through_conv1_and_gather(R):
    """Any bytes in the ring decode without a fault; conv_1 agrees with conv_1 on gather's stacks of the same slots."""
    cap, F, W = 512, 2048, 128
    coded = R.CodedDedupReplay(cap, F, W, 16 * (W + 2 + 8 * 30) * 442)
    _push_both((coded,), None, _stream(400, seed=13), [100] * 4)
    g = torch.Generator(device="cuda"); g.manual_seed(17)
    coded.pool.copy_(torch.randint(0, 256, coded.pool.shape, dtype=torch.uint8, device="cuda", generator=g))
    idx = torch.randint(-3, cap + 3, (512,), device="cuda", generator=g)
    b = coded.gather(idx)
    pack = _packs(R, 2, 32, g)
    for name in ("state", "next_state"):
        yc = R.conv1_fused(coded.frame_source(name), idx, pack, relu=True)
        yg = R.conv1_fused(b[name], None, pack, relu=True)
        for u, v in zip(yc, yg):
            assert torch.equal(u, v)
        gy = torch.randn(512, 32, 20, 20, device="cuda", generator=g)
        assert torch.equal(R.conv1_wgrad(coded.frame_source(name), idx, gy), R.conv1_wgrad(b[name], None, gy))
    torch.cuda.synchronize()


def _learner(apex, coded, B, N):
    cfg = apex.ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                          CUDNN_BENCHMARK=False, FRAME_DEDUP=True, DEDUP_WINDOW=1024, FRAME_CODEC=coded)
    torch.manual_seed(0)
    L = apex.Learner(cfg, connect=None, start_replay=False)
    with torch.no_grad():
        for p in L.target_model.parameters():
            p.add_(0.01 * torch.randn(p.shape, device=p.device))
    return L


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "captured"])
def test_learner_steps_are_bit_identical_to_the_raw_dedup_store(R, graph):
    from distributed_rl_b200 import apex
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B, N = 64, 2048
    recs = _stream(3600, seed=21)
    res = []
    for coded in (False, True):
        L = _learner(apex, coded, B, N)
        for i in range(0, 2400, 300):
            L.memory.push_arrays(*[torch.from_numpy(x[i:i + 300]) for x in recs])
        st = L.memory.store
        assert isinstance(st, R.CodedDedupReplay) == coded
        st.seed(77, 0)
        outs = []
        for k in range(6):
            out = L.fused_step(use_graph=graph)
            outs.append({kk: v.clone() for kk, v in out.items()})
            if k % 2 == 1:                                   # ingest between steps
                i = 2400 + 200 * (k // 2)
                L.memory.push_arrays(*[torch.from_numpy(x[i:i + 200]) for x in recs])
        torch.cuda.synchronize()
        res.append((outs, st.priorities().clone(), [q.detach().clone() for q in L.model.parameters()]))
    (o0, p0, w0), (o1, p1, w1) = res
    for a_, b_ in zip(o0, o1):
        for k in a_:
            assert torch.equal(a_[k], b_[k]), k
    assert torch.equal(p0, p1)
    for u, v in zip(w0, w1):
        assert torch.equal(u, v)


def _stores(R, n, cap, seed):
    s, ns, a, r, d, p = _stream(n, seed=seed)
    raw = R.DedupReplay(cap, 4 * cap, cap // 2)
    coded = R.CodedDedupReplay(cap, 4 * cap, cap // 2, 16 * (4 * cap + 1) * 442)
    for st in (raw, coded):
        for i in range(0, n, 100):
            st.push([torch.from_numpy(x[i:i + 100]) for x in (s, ns, a, r, d)], torch.from_numpy(p[i:i + 100]))
        st.seed(31, 0)
    return raw, coded


def test_serve_fill_and_bound_step_of_a_coded_store_equal_the_raw_store(R):
    from types import SimpleNamespace
    from distributed_rl_b200 import apex
    from distributed_rl_b200.replay_server import ServeRing
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B, slots, steps = 64, 4, 6
    stores = _stores(R, 900, 1024, seed=43)
    rings = [ServeRing.create(st, B, slots) for st in stores]
    try:
        assert bytes(rings[0].layout) == bytes(rings[1].layout)
        for fill in range(slots):
            bufs = []
            for st, ring in zip(stores, rings):
                ring.fill(st, fill, fill + 1, 0.4)
                buf = torch.empty(ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
                ring.take(fill, buf, torch.cuda.current_stream())
                bufs.append(buf)
            torch.cuda.synchronize()
            assert torch.equal(bufs[0], bufs[1]), fill
        res = []
        for ring in rings:
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
                outs.append({kk: v.clone() for kk, v in out.items()})
            torch.cuda.synchronize()
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
