"""GPU tests of the captured Ape-X step on served minibatches (ApexConfig.SERVED_FUSED_STEP).

Kernels: conv_1 forward and weight gradient through a device-resident frame-table entry (the `table` source of
b2rl_frames) against the direct kernels, bit for bit, including an n that the weight gradient splits
over several launches, and a captured graph rebound to other frames.  Bind: b2rl_serve_bind against the slot it
binds.  Learner: a two-process run (the pattern of test_gpu_14_serve.py) whose every bound step is replayed by an
in-process learner, which must end with the same weights, and whose write-backs must all land in the server's
tree, also while the server holds them back."""
import multiprocessing as mp
import pickle
import time

import numpy as np
import pytest

from shared_redis import RedisManager, Shim

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _frames(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, device="cuda", generator=g)


def _pack(n_nets, seed):
    from distributed_rl_b200 import replay as R
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = R.Conv1Pack(n_nets, "cuda")
    for net in range(n_nets):
        p.pack(net, torch.randn(32, 4, 8, 8, device="cuda", generator=g) * 0.05)
    return p


def _table(*tensors):
    return torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device="cuda")


def _gy(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, 32, 20, 20, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("n_nets", [1, 2])
def test_table_variants_equal_the_direct_kernels(relu, n_nets):
    from distributed_rl_b200 import replay as R
    n = 512
    X, pack = _frames(n, 1), _pack(n_nets, 2)
    src = R.BoundFrames(_table(_frames(8, 9), X), 1, n)            # entry 1: the entry offset is honoured
    idx = torch.randint(0, n, (300,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    for rows in (None, idx):
        for a, b in zip(R.conv1_fused(X, rows, pack, relu=relu), R.conv1_fused(src, rows, pack, relu=relu)):
            assert torch.equal(a, b)
    y = R.conv1_fused(X, None, pack, relu=relu)[0]
    gy = _gy(n, 4)
    relu_y = y if relu else None
    assert torch.equal(R.conv1_wgrad(X, None, gy, relu_y=relu_y), R.conv1_wgrad(src, None, gy, relu_y=relu_y))
    gi = _gy(idx.numel(), 5)
    yi = R.conv1_fused(X, idx, pack, relu=True)[0] if relu else None
    assert torch.equal(R.conv1_wgrad(X, idx, gi, relu_y=yi), R.conv1_wgrad(src, idx, gi, relu_y=yi))


def test_table_weight_gradient_split_over_several_launches():
    """n above SMs x 160 frame stacks: b2rl_conv1_wgrad adds each launch's row offset to the table entry on the device."""
    from distributed_rl_b200 import replay as R
    per_launch = torch.cuda.get_device_properties(0).multi_processor_count * 160
    n = per_launch + 257
    X = _frames(n, 6)
    src = R.BoundFrames(_table(X), 0, n)
    gy = _gy(n, 7)
    y = torch.relu(_gy(n, 8))
    a = R.conv1_wgrad(X, None, gy, relu_y=y)
    b = R.conv1_wgrad(src, None, gy, relu_y=y)
    assert torch.equal(a, b)
    # the second launch's rows matter: dropping them changes the gradient
    assert not torch.equal(a, R.conv1_wgrad(X[:per_launch], None, gy[:per_launch], relu_y=y[:per_launch]))
    del X, gy, y
    torch.cuda.empty_cache()


def test_a_captured_graph_follows_the_table():
    """Capture forward + weight gradient over the table bound to X, rebind it to Y, replay: the eager results on Y."""
    from distributed_rl_b200 import replay as R
    n = 512
    X, Y, pack = _frames(n, 10), _frames(n, 11), _pack(2, 12)
    table = _table(X)
    src = R.BoundFrames(table, 0, n)
    out = torch.empty((2, n, 20, 20, 32), device="cuda")
    gw = torch.empty(32, 4, 8, 8, device="cuda")
    gy = _gy(n, 13)

    def step():
        y = R.conv1_fused(src, None, pack, relu=True, out=out)[0]
        R.conv1_wgrad(src, None, gy, out=gw, relu_y=y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                     # smem attributes and the wgrad workspace outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    table.copy_(_table(Y))
    g.replay()
    torch.cuda.synchronize()
    ref = R.conv1_fused(Y, None, pack, relu=True)
    assert torch.equal(out[0], ref[0].permute(0, 2, 3, 1)) and torch.equal(out[1], ref[1].permute(0, 2, 3, 1))
    assert torch.equal(gw, R.conv1_wgrad(Y, None, gy, relu_y=ref[0]))
    assert not torch.equal(gw, R.conv1_wgrad(X, None, gy, relu_y=R.conv1_fused(X, None, pack, relu=True)[0]))


def test_bind_copies_the_slot_and_points_the_table_at_its_frames():
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.replay_server import ServeRing
    B = 48
    st = R.DeviceReplay(64, R.APEX_FIELDS, "cuda:0")
    st.fill_hash(60, seed=3)
    st.build(torch.rand(60, generator=torch.Generator().manual_seed(4)).cuda() + 0.05)
    ring = ServeRing.create(st, B, 2)
    try:
        st.seed(5, 0)
        ring.fill(st, 1, 777, 0.4)
        cur = dict(R.alloc_rows(R.APEX_FIELDS, B, "cuda:0", ("action", "reward", "done")),
                   idx=torch.empty(B, dtype=torch.int64, device="cuda"),
                   w=torch.empty(B, dtype=torch.float32, device="cuda"),
                   header=torch.zeros(2, dtype=torch.int64, device="cuda"))
        table = torch.zeros(2, dtype=torch.int64, device="cuda")
        frames = {"state": R.BoundFrames(table, 0, B), "next_state": R.BoundFrames(table, 1, B)}
        ptrs = ring.slot_ptrs(1)[0]
        ring.bind(ptrs[0], R.APEX_FIELDS, cur, frames, torch.cuda.current_stream())
        buf = torch.empty(ring.layout.slot_bytes, dtype=torch.uint8, device="cuda")
        ring.take(1, buf, torch.cuda.current_stream())
        torch.cuda.synchronize()
        L = ring.layout

        def view(off, nbytes):
            return buf[off:off + nbytes]
        assert cur["header"].tolist() == [777, B]
        assert torch.equal(cur["header"].view(torch.uint8), view(0, 16))
        assert torch.equal(cur["idx"].view(torch.uint8), view(L.idx_off, 8 * B))
        assert torch.equal(cur["w"].view(torch.uint8), view(L.w_off, 4 * B))
        for i, f in enumerate(R.APEX_FIELDS):
            if f.name in cur:
                assert torch.equal(cur[f.name].view(torch.uint8).reshape(-1), view(L.field_off[i], B * f.nbytes)), f.name
        assert table.tolist() == [ptrs[3], ptrs[4]]      # state, next_state rows inside the slot
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


# ---- two processes --------------------------------------------------------------------------------------------------
def _server_main(proxy, cfg_kw, stop, out, hold):
    """The replay server: serve until `stop`, then report the tree's leaves and free the ring.  `hold`: update slots
    are applied only once the server has handed out that many fills, so the learner's write-backs queue up."""
    from distributed_rl_b200 import apex
    from distributed_rl_b200.replay_server import DeviceReplayServer
    srv = DeviceReplayServer(apex.ApexConfig(**cfg_kw), Shim(proxy), slots=2)
    srv.store.seed(4242, 0)
    while not stop.is_set():
        data = srv._ingest_experience()
        busy = len(data) + srv.slots.collect_releases(srv._wait_released)
        if srv.slots.seq >= hold:
            busy += srv.slots.apply_updates(srv._apply)
        busy += srv.slots.fill_free(srv._fill) if srv._can_fill() else 0
        srv._publish_stats(bool(data))
        if not busy:
            time.sleep(0.0005)
    torch.cuda.synchronize()
    leaves = srv.store.priorities(0, srv.cfg.REPLAY_MEMORY_LEN).cpu().numpy()
    out.put((leaves, srv.close(timeout=60)))


def _apex_rec(rng, prio):
    return [rng.integers(0, 256, (4, 84, 84), dtype=np.uint8), int(rng.integers(6)), float(rng.standard_normal()),
            rng.integers(0, 256, (4, 84, 84), dtype=np.uint8), bool(rng.random() < 0.3), float(prio)]


@pytest.mark.parametrize("server_device,hold", [("cuda:0", 0), ("cuda:1", 0), ("cuda:0", 10)])
def test_served_fused_step_round_trip(server_device, hold):
    if torch.cuda.device_count() < int(server_device[-1]) + 1:
        pytest.skip("needs two GPUs")
    from distributed_rl_b200 import apex
    from distributed_rl_b200.replay_server import DeviceReplayClient
    N, B, steps, log_every = 64, 32, 20, 10
    base = dict(BATCHSIZE=B, REPLAY_MEMORY_LEN=128, BUFFER_SIZE=40, CUDNN_BENCHMARK=False)
    ctx = mp.get_context("spawn")
    mgr = RedisManager(ctx=ctx)
    mgr.start()
    child, stop, client = None, ctx.Event(), None
    try:
        proxy = mgr.Redis()
        conn = Shim(proxy)
        out = ctx.Queue()
        child = ctx.Process(target=_server_main,
                            args=(proxy, dict(base, LEARNER_DEVICE=server_device), stop, out, hold))
        child.start()
        rng = np.random.default_rng(0)
        recs = [_apex_rec(rng, 0.25 + 0.5 * rng.random()) for _ in range(N)]
        blobs = [pickle.dumps(r) for r in recs]
        conn.rpush("experience", *blobs)
        client = DeviceReplayClient(apex.ApexConfig(**base, LEARNER_DEVICE="cuda:0"), conn, timeout=180.0)
        bound, updates, queued = [], [], []
        acquire, update = client.acquire, client.update

        def rec_acquire(cur, frames):
            d = acquire(cur, frames)
            if d is not None:
                bound.append((d, {k: v.clone() for k, v in cur.items()}))
            return d

        def rec_update(idx, vals):
            updates.append((idx.clone(), vals.clone()))
            update(idx, vals)
            queued.append(len(client._pending))
        client.acquire, client.update = rec_acquire, rec_update
        torch.manual_seed(0)
        L = apex.Learner(apex.ApexConfig(**base, LEARNER_DEVICE="cuda:0", SERVED_FUSED_STEP=True), connect=conn,
                         start_replay=False, memory=client)
        assert L.run(max_steps=steps, log_every=log_every) == steps
        torch.cuda.synchronize()
        assert L._graph is not None                     # steps after the warm-up replayed the captured graph
        assert len(bound) == steps                      # warm-up steps included
        assert len(updates) == steps - steps // log_every   # the eviction steps skip their write-back
        if hold:
            assert max(queued) >= 2                     # several graph write-backs waited at once
        # every served header is its descriptor's
        seqs = [d[1] for d, _ in bound]
        for (k, seq, n), b in bound:
            assert n == B and b["header"].tolist() == [seq, B]
        assert seqs == sorted(seqs) and len(set(seqs)) == steps
        # the same records in a ring of the same capacity: the slot ids match
        torch.manual_seed(0)
        L2 = apex.Learner(apex.ApexConfig(**base, LEARNER_DEVICE="cuda:0"), connect=None, start_replay=False)
        L2.memory.push_records(blobs)
        st = L2.memory.store
        s2 = L2._fused_state()
        batched = L2.cfg.PARALLEL_FORWARDS and L2.cfg.BATCHED_ONLINE
        L2.optim.zero_grad(set_to_none=False)
        for _, b in bound:
            g = st.gather(b["idx"], st.alloc_batch(B, ("action", "reward", "done")))
            for name in ("action", "reward", "done"):          # the bound scalars are the records at idx
                assert torch.equal(b[name], g[name]), name
            assert torch.isfinite(b["w"]).all() and (b["w"] > 0).all() and (b["w"] <= 1).all()
            L2._pack_weights()
            L2._forward_backward_fused(b["idx"], b["action"] if batched else b["action"].to(torch.int64),
                                       b["reward"], b["done"], b["w"], prepacked=True, early_update=True)
            L2.step()
        assert s2.pack1 is not None
        torch.cuda.synchronize()
        for (name, p1), p2 in zip(L.model.state_dict().items(), L2.model.state_dict().values()):
            assert torch.equal(p1, p2), name
        # every write-back lands in the server's tree (last writer wins)
        t0 = time.time()
        while len(client.slots.upd_free) < client.ring.layout.slots or client._pending:
            assert time.time() - t0 < 60, "update slots not handed back"
            client.slots.poll()
            client._flush_updates()
            time.sleep(0.005)
        want = np.zeros(128, np.float32)
        want[:N] = np.float32([r[5] for r in recs])
        for i, v in updates:
            want[i.cpu().numpy()] = v.cpu().numpy()
        client.close()
        client = None
        stop.set()
        leaves, freed = out.get(timeout=120)
        np.testing.assert_array_equal(leaves, want)
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
