"""GPU tests of the device serve ring (replay_server.DeviceReplayServer / DeviceReplayClient, csrc/serve.cu).

One process: b2rl_serve_fill against b2rl_tree_sample_fetch + b2rl_replay_gather from the same RNG state (bit for
bit, RNG counter included) and against the numpy oracle on dyadic priorities.

Two processes: the server runs in a `spawn` child (cudaIpcOpenMemHandle cannot map a handle into the process that
exported it); the control plane is a FakeRedis hosted by a multiprocessing manager, whose pipelines the client shim
builds locally and executes atomically in the manager."""
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


def _slot_views(layout, buf):
    """header, idx, w and the Ape-X fields of a copied-out minibatch slot."""
    from distributed_rl_b200 import replay as R
    B = layout.batch

    def view(off, nbytes, dtype, shape):
        return buf[off:off + nbytes].view(dtype).view(shape)
    out = {f.name: view(layout.field_off[i], B * f.nbytes, f.dtype, (B,) + tuple(f.shape))
           for i, f in enumerate(R.APEX_FIELDS)}
    return view(0, 16, torch.int64, (2,)), view(layout.idx_off, 8 * B, torch.int64, (B,)), \
        view(layout.w_off, 4 * B, torch.float32, (B,)), out


def _take(ring, k):
    buf = torch.empty(ring.layout.slot_bytes, dtype=torch.uint8, device=ring.device)
    ring.take(k, buf, torch.cuda.current_stream(ring.device))
    return _slot_views(ring.layout, buf)


def _fetch_and_gather(st, B, beta):
    idx = torch.empty(B, dtype=torch.int64, device=st.device)
    w = torch.empty(B, dtype=torch.float32, device=st.device)
    small = st.alloc_batch(B, ("action", "reward", "done"))
    st.sample_fetch(B, beta, idx, w, small)
    big = st.gather(idx, st.alloc_batch(B, ("state", "next_state")))
    return idx, w, dict(small, **big)


def _check_fill_equals_fetch_gather(st, B, seed, counter, beta=0.4):
    from distributed_rl_b200.replay_server import ServeRing
    ring = ServeRing.create(st, B, 2)
    try:
        st.seed(seed, counter)
        idx, w, ref = _fetch_and_gather(st, B, beta)
        idx_next, w_next, _ = _fetch_and_gather(st, B, beta)          # what the advanced counter draws next
        st.seed(seed, counter)
        ring.fill(st, 1, 12345, beta)
        idx2, w2, _ = _fetch_and_gather(st, B, beta)                   # the fill advanced the counter by B as well
        hdr, sidx, sw, sb = _take(ring, 1)
        torch.cuda.synchronize()
        assert hdr.tolist() == [12345, B]
        assert torch.equal(sidx, idx) and torch.equal(sw.view(torch.int32), w.view(torch.int32))
        for name in ("state", "next_state", "action", "reward", "done"):     # as bytes: hashed floats may be NaN
            assert torch.equal(sb[name].view(torch.uint8), ref[name].view(torch.uint8)), name
        assert torch.equal(idx2, idx_next) and torch.equal(w2, w_next)
        # slot 0 was never filled: its header is still zero
        assert _take(ring, 0)[0].tolist() == [0, 0]
        return idx
    finally:
        torch.cuda.synchronize()
        ring.close()


def test_fill_equals_fetch_plus_gather_small_store_with_duplicates():
    from distributed_rl_b200 import replay as R
    st = R.DeviceReplay(40, R.APEX_FIELDS, "cuda:0")
    st.fill_hash(37, seed=5)
    p = torch.rand(40, generator=torch.Generator().manual_seed(1)) + 0.05
    p[:3] *= 40.0                                      # three heavy slots: most draws repeat
    st.build(p[:37].cuda())
    # B = 2048: 16 draws x 2 chunks per CTA, more items than shared-memory stages, so the ring's stages are refilled
    for B, seed, counter in ((96, 7, 0), (96, 7, 123456), (96, 0xFFFF_FFFF_1234, 2 ** 40), (2048, 3, 99)):
        idx = _check_fill_equals_fetch_gather(st, B, seed, counter)
        assert idx.unique().numel() < idx.numel()     # duplicate draws were copied too
    st.close()


def test_fill_equals_fetch_plus_gather_full_store_b512():
    from distributed_rl_b200 import replay as R
    free, _ = torch.cuda.mem_get_info()
    if free < 64 * 2 ** 30:
        pytest.skip("needs a 2^20-slot store (59 GB) on one device")
    n = 2 ** 20
    st = R.DeviceReplay(n, R.APEX_FIELDS, "cuda:0")
    st.fill_hash(n, seed=0xB200)
    st.build(torch.rand(n, generator=torch.Generator().manual_seed(2)).cuda() + 1e-3)
    _check_fill_equals_fetch_gather(st, 512, 99, 7)
    st.close()
    torch.cuda.empty_cache()


def test_fill_matches_the_oracle_on_dyadic_priorities():
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.replay_server import ServeRing
    from oracle import oracle as O
    n, B = 4096, 256
    rng = np.random.default_rng(3)
    p = (2.0 ** rng.integers(-6, 3, n)).astype(np.float32)       # dyadic: every fp32 partial sum is exact
    st = R.DeviceReplay(n, R.APEX_FIELDS, "cuda:0")
    st.fill_hash(n, seed=11)
    st.build(torch.from_numpy(p).cuda())
    ring = ServeRing.create(st, B, 1)
    st.seed(21, 500)
    ring.fill(st, 0, 1, 0.4)
    _, sidx, sw, sb = _take(ring, 0)
    u = st.philox_uniforms(21, 500, B).cpu().numpy()
    t = O.SumTreeOracle(n)
    t.build(p)
    oidx, _ = t.sample(u)
    ow, _, _ = O.is_weights(p[oidx], t.total, t.min_priority, n, 0.4)
    assert np.array_equal(sidx.cpu().numpy(), oidx)
    assert np.allclose(sw.cpu().numpy(), ow, rtol=2.4e-7)
    want = O.hash_rows(0, oidx, R.FRAME_STACK_BYTES, 11)
    assert np.array_equal(sb["state"].reshape(B, -1).cpu().numpy(), want)
    torch.cuda.synchronize()
    ring.close()
    st.close()


# ---- two processes --------------------------------------------------------------------------------------------------
def _server_main(proxy, cfg_kw, stop, out):
    """The replay server process: serve until `stop`, then report the tree's leaves and free the ring."""
    from distributed_rl_b200 import apex
    from distributed_rl_b200.replay_server import DeviceReplayServer
    srv = DeviceReplayServer(apex.ApexConfig(**cfg_kw), Shim(proxy), slots=3)
    srv.store.seed(4242, 0)
    while not stop.is_set():
        st = srv.serve_once()
        if not (st["ingested"] or st["filled"] or st["released"] or st["updates_applied"]):
            time.sleep(0.0005)
    torch.cuda.synchronize()
    leaves = srv.store.priorities(0, srv.cfg.REPLAY_MEMORY_LEN).cpu().numpy()
    out.put((leaves, srv.close(timeout=60)))     # frees the ring once the learner has detached


def _apex_rec(rng, prio):
    return [rng.integers(0, 256, (4, 84, 84), dtype=np.uint8), int(rng.integers(6)), float(rng.standard_normal()),
            rng.integers(0, 256, (4, 84, 84), dtype=np.uint8), bool(rng.random() < 0.3), float(prio)]


@pytest.mark.parametrize("server_device", ["cuda:0", "cuda:1"])
def test_two_process_round_trip(server_device):
    if torch.cuda.device_count() < int(server_device[-1]) + 1:
        pytest.skip("needs two GPUs")
    from distributed_rl_b200 import apex
    from distributed_rl_b200.replay_server import DeviceReplayClient
    N, B, steps = 64, 32, 20
    base = dict(BATCHSIZE=B, REPLAY_MEMORY_LEN=128, BUFFER_SIZE=40, CUDNN_BENCHMARK=False)
    ctx = mp.get_context("spawn")
    mgr = RedisManager(ctx=ctx)
    mgr.start()
    child, stop, client = None, ctx.Event(), None
    try:
        proxy = mgr.Redis()
        conn = Shim(proxy)
        out = ctx.Queue()
        child = ctx.Process(target=_server_main, args=(proxy, dict(base, LEARNER_DEVICE=server_device), stop, out))
        child.start()
        rng = np.random.default_rng(0)
        recs = [_apex_rec(rng, 0.25 + 0.5 * rng.random()) for _ in range(N)]
        conn.rpush("experience", *[pickle.dumps(r) for r in recs])
        client = DeviceReplayClient(apex.ApexConfig(**base, LEARNER_DEVICE="cuda:0"), conn, timeout=180.0)
        served, updates = [], []
        sample, update = client.sample, client.update

        def rec_sample():
            b = sample()
            if b is not False:
                served.append(([t.clone() for t in b], client.last_served, client.last_header.clone()))
            return b

        def rec_update(idx, vals):
            updates.append((torch.as_tensor(idx).clone(), torch.as_tensor(vals).clone()))
            update(idx, vals)
        client.sample, client.update = rec_sample, rec_update
        from distributed_rl_b200 import replay_server as RS
        conn.set("Start", b"stale-from-a-previous-run")
        torch.manual_seed(0)
        L = apex.Learner(apex.ApexConfig(**base, LEARNER_DEVICE="cuda:0"), connect=conn, start_replay=False,
                         memory=client)
        # the start-up wipe drops stale keys but not the handshake the client and the server already set up
        assert conn.get("Start") is None
        assert conn.get(RS.CLIENT_KEY) is not None and conn.get(RS.RING_KEY) is not None
        assert L.run(max_steps=steps) == steps
        torch.cuda.synchronize()
        assert pickle.loads(conn.get("Start")) is True and conn.get("state_dict") is not None
        assert len(served) == steps and len(updates) == steps
        # (a) every served minibatch is the pushed records at its idx, and its header is its descriptor's
        seqs = []
        for (s, a, r, ns, d, w, idx), (k, seq, n), hdr in served:
            ii = idx.cpu().numpy()
            assert n == B and hdr.tolist() == [seq, B]
            seqs.append(seq)
            np.testing.assert_array_equal(s.cpu().numpy(), np.stack([recs[i][0] for i in ii]))
            np.testing.assert_array_equal(ns.cpu().numpy(), np.stack([recs[i][3] for i in ii]))
            np.testing.assert_array_equal(a.cpu().numpy(), [recs[i][1] for i in ii])
            np.testing.assert_array_equal(r.cpu().numpy(), np.float32([recs[i][2] for i in ii]))
            np.testing.assert_array_equal(d.cpu().numpy(), [recs[i][4] for i in ii])
            assert torch.isfinite(w).all() and (w > 0).all() and (w <= 1).all()
        assert seqs == sorted(seqs) and len(set(seqs)) == steps
        # (c) the same learner fed the same minibatches directly ends with the same weights, bit for bit
        torch.manual_seed(0)
        L2 = apex.Learner(apex.ApexConfig(**base, LEARNER_DEVICE="cuda:0"), connect=None, start_replay=False)
        for b, _, _ in served:
            L2.train(b)
        torch.cuda.synchronize()
        for (name, p1), p2 in zip(L.model.state_dict().items(), L2.model.state_dict().values()):
            assert torch.equal(p1, p2), name
        # (b) every write-back lands in the server's tree (last writer wins)
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
        assert freed                                   # the server saw SERVE_DETACHED before freeing the ring
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
