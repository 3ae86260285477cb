"""GPU tests of the stand-alone replay mode for R2D2 (replay_server with an R2D2Config, csrc/serve.cu).

One process: b2rl_serve_fill of the R2D2 sequence record (frame rows and LSTM state as TMA bulk rows, the 80-step
action / reward rows copied by the fill's other warps, notdone as a scalar) against b2rl_tree_sample_fetch +
b2rl_replay_gather from the same RNG state, bit for bit, at batch sizes below and above the SM count; and against the
numpy oracle on dyadic priorities.

Two processes: a DeviceReplayServer in a `spawn` child feeds `r2d2.Learner(memory=DeviceReplayClient(...)).run()`
through the ring, over a FakeRedis hosted by a multiprocessing manager (as test_gpu_14_serve.py).  The Redis-protocol
pair ReplayServer -> Replay_Server -> r2d2.Learner.train runs in one process on a FakeRedis."""
import multiprocessing as mp
import pickle
import time

import numpy as np
import pytest

from shared_redis import RedisManager, Shim
from test_wire_cpu import _r2d2_record

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _take(ring, k, fields):
    """header, idx, w and the fields of minibatch slot k, copied out of the ring."""
    L, B = ring.layout, ring.layout.batch
    buf = torch.empty(L.slot_bytes, dtype=torch.uint8, device=ring.device)
    ring.take(k, buf, torch.cuda.current_stream(ring.device))

    def view(off, nbytes, dtype, shape):
        return buf[off:off + nbytes].view(dtype).view(shape)
    out = {f.name: view(L.field_off[i], B * f.nbytes, f.dtype, (B,) + tuple(f.shape)) for i, f in enumerate(fields)}
    return view(0, 16, torch.int64, (2,)), view(L.idx_off, 8 * B, torch.int64, (B,)), \
        view(L.w_off, 4 * B, torch.float32, (B,)), out


BIG = ("state", "action", "reward", "h0", "h1")


def _fetch_and_gather(st, B, beta):
    idx = torch.empty(B, dtype=torch.int64, device=st.device)
    w = torch.empty(B, dtype=torch.float32, device=st.device)
    small = st.alloc_batch(B, ("notdone",))
    st.sample_fetch(B, beta, idx, w, small)
    big = st.gather(idx, st.alloc_batch(B, BIG))
    return idx, w, dict(small, **big)


@pytest.mark.parametrize("B", [1, 16, 32, 64, 200])
def test_r2d2_fill_equals_fetch_plus_gather_with_duplicates(B):
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.replay_server import ServeRing
    fields = R.r2d2_fields(80)
    st = R.DeviceReplay(40, fields, "cuda:0")
    st.fill_hash(37, seed=5)
    p = torch.rand(40, generator=torch.Generator().manual_seed(1)) + 0.05
    p[:3] *= 40.0                                      # three heavy slots: most draws repeat
    st.build(p[:37].cuda())
    ring = ServeRing.create(st, B, 2)
    try:
        for seed, counter in ((7, 0), (0xFFFF_FFFF_1234, 2 ** 40)):
            st.seed(seed, counter)
            idx, w, ref = _fetch_and_gather(st, B, 0.4)
            idx_next, w_next, _ = _fetch_and_gather(st, B, 0.4)      # what the advanced counter draws next
            st.seed(seed, counter)
            ring.fill(st, 1, 777, 0.4)
            idx2, w2, _ = _fetch_and_gather(st, B, 0.4)               # the fill advanced the counter by B as well
            hdr, sidx, sw, sb = _take(ring, 1, fields)
            torch.cuda.synchronize()
            assert hdr.tolist() == [777, B]
            assert torch.equal(sidx, idx) and torch.equal(sw.view(torch.int32), w.view(torch.int32))
            for f in fields:                                          # as bytes: hashed floats may be NaN
                assert torch.equal(sb[f.name].view(torch.uint8), ref[f.name].view(torch.uint8)), f.name
            assert torch.equal(idx2, idx_next) and torch.equal(w2, w_next)
            if B >= 16:
                assert idx.unique().numel() < idx.numel()             # duplicate draws were copied too
        assert _take(ring, 0, fields)[0].tolist() == [0, 0]           # slot 0 was never filled
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


def test_r2d2_fill_matches_the_oracle_on_dyadic_priorities():
    """T = 4 keeps a 4096-sequence store small; action / reward are then 16-byte small rows."""
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.replay_server import ServeRing
    from oracle import oracle as O
    n, B, T = 4096, 64, 4
    fields = R.r2d2_fields(T)
    rng = np.random.default_rng(3)
    p = (2.0 ** rng.integers(-6, 3, n)).astype(np.float32)       # dyadic: every fp32 partial sum is exact
    st = R.DeviceReplay(n, fields, "cuda:0")
    st.fill_hash(n, seed=11)
    st.build(torch.from_numpy(p).cuda())
    ring = ServeRing.create(st, B, 1)
    st.seed(21, 500)
    ring.fill(st, 0, 1, 0.4)
    _, sidx, sw, sb = _take(ring, 0, fields)
    u = st.philox_uniforms(21, 500, B).cpu().numpy()
    t = O.SumTreeOracle(n)
    t.build(p)
    oidx, _ = t.sample(u)
    ow, _, _ = O.is_weights(p[oidx], t.total, t.min_priority, n, 0.4)
    assert np.array_equal(sidx.cpu().numpy(), oidx)
    assert np.allclose(sw.cpu().numpy(), ow, rtol=2.4e-7)
    for i, f in enumerate(fields):
        got = sb[f.name].reshape(B, -1).view(torch.uint8).cpu().numpy()
        assert np.array_equal(got, O.hash_rows(i, oidx, f.nbytes, 11)), f.name
    torch.cuda.synchronize()
    ring.close()
    st.close()


# ---- two processes --------------------------------------------------------------------------------------------------
def _server_main(proxy, cfg_kw, stop, out):
    """The replay server process: serve until `stop`, then report the tree's leaves and free the ring."""
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200.replay_server import DeviceReplayServer
    srv = DeviceReplayServer(r2d2.R2D2Config(**cfg_kw), Shim(proxy), slots=3)
    srv.store.seed(4242, 0)
    while not stop.is_set():
        st = srv.serve_once()
        if not (st["ingested"] or st["filled"] or st["released"] or st["updates_applied"]):
            time.sleep(0.0005)
    torch.cuda.synchronize()
    leaves = srv.store.priorities(0, srv.cfg.REPLAY_MEMORY_LEN).cpu().numpy()
    out.put((leaves, srv.close(timeout=60)))


def _clone(b):
    (h0, h1), rest = b[0], b[1:]
    return [(h0.clone(), h1.clone())] + [t.clone() for t in rest]


def _check_served(b, cols, B):
    """A served minibatch [(h0, h1), s, a, r, notdone, w, idx] holds the pushed records at its idx."""
    (h0, h1), s, a, r, nd, w, idx = b
    ii = torch.as_tensor(idx).cpu().numpy()
    assert h0.shape == (1, B, 512) and h1.shape == (1, B, 512)
    for got, want in ((s, cols[0]), (a, cols[1]), (r, cols[2]), (h0[0], cols[3]), (h1[0], cols[4]), (nd, cols[5])):
        np.testing.assert_array_equal(torch.as_tensor(got).cpu().numpy(), want[ii])
    w = torch.as_tensor(w)
    assert torch.isfinite(w).all() and (w > 0).all() and (w <= 1).all()


def test_two_process_r2d2_round_trip():
    from distributed_rl_b200 import r2d2, wire
    from distributed_rl_b200 import replay_server as RS
    N, B, steps, T = 40, 4, 10, 80
    base = dict(BATCHSIZE=B, REPLAY_MEMORY_LEN=64, BUFFER_SIZE=16, LEARNER_DEVICE="cuda:0")
    ctx = mp.get_context("spawn")
    mgr = RedisManager(ctx=ctx)
    mgr.start()
    child, stop, client = None, ctx.Event(), None
    try:
        proxy = mgr.Redis()
        conn = Shim(proxy)
        out = ctx.Queue()
        child = ctx.Process(target=_server_main, args=(proxy, base, stop, out))
        child.start()
        rng = np.random.default_rng(0)
        recs = [_r2d2_record(rng, T, bool(i % 5 == 0)) for i in range(N)]
        cols, prios = wire.decode_r2d2(recs, T)
        conn.rpush("experience", *[pickle.dumps(r) for r in recs])
        client = RS.DeviceReplayClient(r2d2.R2D2Config(**base), conn, timeout=180.0)
        served, updates = [], []
        sample, update = client.sample, client.update

        def rec_sample():
            b = sample()
            if b is not False:
                served.append((_clone(b), client.last_served, client.last_header.clone()))
            return b

        def rec_update(idx, vals):
            updates.append((torch.as_tensor(idx).clone(), torch.as_tensor(vals).clone()))
            update(idx, vals)
        client.sample, client.update = rec_sample, rec_update
        conn.set("Start", b"stale-from-a-previous-run")
        torch.manual_seed(0)
        L = r2d2.Learner(r2d2.R2D2Config(**base), connect=conn, start_replay=False, memory=client)
        assert L.memory is client
        assert conn.get("Start") is None                 # the start-up wipe drops stale keys ...
        assert conn.get(RS.CLIENT_KEY) is not None and conn.get(RS.RING_KEY) is not None   # ... not the handshake
        assert L.run(max_steps=steps, log_every=5) == steps
        torch.cuda.synchronize()
        assert pickle.loads(conn.get("Start")) is True
        # steps 5 and 10 raise the eviction request through the client's lock and skip their write-back
        assert len(served) == steps and len(updates) == steps - 2
        assert pickle.loads(conn.get("FLAG_REMOVE")) is True
        seqs = []
        for b, (k, seq, n), hdr in served:
            assert n == B and hdr.tolist() == [seq, B]
            seqs.append(seq)
            _check_served(b, cols, B)
        assert seqs == sorted(seqs) and len(set(seqs)) == steps
        # the same learner fed the same minibatches directly ends with the same weights, bit for bit
        torch.manual_seed(0)
        L2 = r2d2.Learner(r2d2.R2D2Config(**base), connect=None, start_replay=False)
        for b, _, _ in served:
            L2.train(b)
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
        want = np.zeros(64, np.float32)
        want[:N] = prios
        for i, v in updates:
            want[i.cpu().numpy()] = v.cpu().numpy()
        client.close()
        client = None
        stop.set()
        leaves, freed = out.get(timeout=120)
        np.testing.assert_array_equal(leaves, want)
        assert freed                                     # the server saw SERVE_DETACHED before freeing the ring
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


def test_redis_protocol_pair_feeds_the_r2d2_learner():
    """ReplayServer -> pickled `BATCH` -> Replay_Server -> r2d2.Learner.train, and the learner's priorities back
    through `update` into the server's tree."""
    from fake_redis import FakeRedis
    from distributed_rl_b200 import r2d2, wire
    from distributed_rl_b200.replay_server import Replay_Server, ReplayServer
    N, B, T = 24, 4, 80
    cfg = r2d2.R2D2Config(BATCHSIZE=B, REPLAY_MEMORY_LEN=32, BUFFER_SIZE=8, LEARNER_DEVICE="cuda:0")
    conn = FakeRedis()
    srv = ReplayServer(cfg, conn)
    srv.store.seed(99, 0)
    rng = np.random.default_rng(1)
    recs = [_r2d2_record(rng, T, bool(i % 4 == 0)) for i in range(N)]
    cols, prios = wire.decode_r2d2(recs, T)
    conn.rpush("experience", *[pickle.dumps(r) for r in recs])
    st = srv.serve_once()
    assert st["ingested"] == N and st["batches_queued"] == 8 and pickle.loads(conn.get("FLAG_BATCH")) is False
    cli = Replay_Server(cfg, conn)
    cli.poll_once()
    assert len(cli.deque) == 8
    torch.manual_seed(0)
    L = r2d2.Learner(cfg, connect=None, start_replay=False)
    idx_all, prio_all = [], []
    while (b := cli.sample()) is not False:
        _check_served(b, cols, B)
        info, prio, idx = L.train(b)
        assert torch.isfinite(prio).all() and torch.isfinite(info["p_norm"])
        cli.update(idx, prio)
        idx_all += torch.as_tensor(idx).tolist()
        prio_all.append(prio.detach().cpu().numpy())
    assert len(idx_all) == 8 * B
    # what poll_once sends once more than 1000 write-backs are queued
    conn.rpush("update", pickle.dumps((cli.idx[:], np.concatenate(cli.vals, 0))))
    assert srv.update() == 8 * B
    torch.cuda.synchronize()
    want = np.zeros(32, np.float32)
    want[:N] = prios
    for i, v in zip(idx_all, np.concatenate(prio_all)):
        want[i] = v
    np.testing.assert_array_equal(srv.store.priorities(0, 32).cpu().numpy(), want)
    srv.store.close()
