"""GPU tests of the stand-alone replay mode for IMPALA (replay_server with an ImpalaConfig, b2rl_serve_fill_uniform in
csrc/serve.cu).

One process: the fill's draw against its numpy restatement (tests/uniform_oracle.py) bit for bit on a wrapped ring, at
batch sizes below and above the SM count, with the Philox counter advancing by B; every field of the slot against
DeviceReplay.gather of the drawn slots, transposed to time-major, byte for byte; a chi-square test of the marginal
counts; and the refusal of a batch larger than the stored records.

Two processes: a DeviceReplayServer(ImpalaConfig) in a `spawn` child ingests `trajectory` records and feeds
`impala.Learner(memory=DeviceReplayClient(...)).run()` through the ring, over a FakeRedis hosted by a multiprocessing
manager (as test_gpu_16_r2d2_serve.py)."""
import multiprocessing as mp
import pickle

import numpy as np
import pytest

from shared_redis import RedisManager, Shim
from uniform_oracle import uniform_draw

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _store(T, capacity, pushes, evict=0, seed=0):
    """An IMPALA store on cuda:0 after `pushes` rollouts of random bytes (pushed in chunks, so the ring wraps), then
    `evict` of the oldest dropped."""
    from distributed_rl_b200 import replay as R
    st = R.DeviceReplay(capacity, R.impala_fields(T), "cuda:0")
    g = torch.Generator(device="cuda:0").manual_seed(seed)
    done = 0
    while done < pushes:
        n = min(37, pushes - done)
        cols = [torch.randint(0, 256, (n * f.nbytes,), dtype=torch.uint8, device="cuda:0", generator=g)
                .view(f.dtype).view((n,) + tuple(f.shape)) for f in st.fields]
        st.push(cols, torch.ones(n))
        done += n
    if evict:
        st.evict(evict)
    torch.cuda.synchronize()
    return st


def _take(ring, k, fields):
    """header, idx, w and the time-major fields of minibatch slot k, copied out of the ring."""
    L, B = ring.layout, ring.layout.batch
    buf = torch.empty(L.slot_bytes, dtype=torch.uint8, device=ring.device)
    ring.take(k, buf, torch.cuda.current_stream(ring.device))

    def view(off, nbytes, dtype, shape):
        return buf[off:off + nbytes].view(dtype).view(shape)
    out = {f.name: view(L.field_off[i], B * f.nbytes, f.dtype, (f.shape[0], B) + tuple(f.shape[1:]) if f.shape else (B,))
           for i, f in enumerate(fields)}
    return view(0, 16, torch.int64, (2,)), view(L.idx_off, 8 * B, torch.int64, (B,)), view(L.w_off, 4 * B, torch.uint8,
                                                                                           (4 * B,)), out


@pytest.mark.parametrize("B,T,cap,pushes,evict", [(1, 2, 256, 300, 20), (16, 2, 256, 300, 20), (32, 20, 64, 100, 0),
                                                   (200, 2, 256, 300, 20)])
def test_uniform_fill_equals_the_oracle_and_the_time_major_gather(B, T, cap, pushes, evict):
    from distributed_rl_b200.replay_server import ServeRing
    st = _store(T, cap, pushes, evict)
    size, _, head = st._sizes()
    assert size == min(cap, pushes) - evict and (head - size) % cap != 0      # the valid region wraps
    ring = ServeRing.create(st, B, 2)
    try:
        for seed, counter in ((7, 0), (0xFFFF_FFFF_1234, 2 ** 40)):
            st.seed(seed, counter)
            ring.fill_uniform(st, 1, 777, T)
            ring.fill_uniform(st, 0, 778, T)                 # the counter advanced by B
            for k, seq, off in ((1, 777, 0), (0, 778, B)):
                hdr, idx, w, got = _take(ring, k, st.fields)
                torch.cuda.synchronize()
                assert hdr.tolist() == [seq, B]
                want = uniform_draw(seed, counter + off, B, size, cap, head)
                assert np.array_equal(idx.cpu().numpy(), want)
                assert not w.any()                           # no IS weights: w is never written
                ref = st.gather(idx)
                for f in st.fields:
                    r = ref[f.name]
                    r = r.transpose(0, 1) if f.shape else r  # (B, T(+1), ...) -> time-major
                    assert torch.equal(got[f.name].reshape(-1).view(torch.uint8),
                                       r.contiguous().reshape(-1).view(torch.uint8)), f.name
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


def test_uniform_fill_marginals_pass_a_chi_square_test():
    """4000 fills of 32 from 1000 rollouts (not a power of two: the Feistel domain is 1024 and the cycle-walk runs)."""
    from scipy import stats
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.replay_server import ServeRing
    st = _store(1, 1000, 1000)
    ring = ServeRing.create(st, 32, 1)
    st.seed(2024, 0)
    idx_ptr = ring.slot_ptrs(0)[0][1]
    with torch.cuda.device(st.device):
        idx = torch.as_tensor(R._CudaView(idx_ptr, (32,), "<i8", ring), device=st.device)
    draws = torch.empty(4000, 32, dtype=torch.int64, device=st.device)
    for f in range(4000):
        ring.fill_uniform(st, 0, f + 1, 1)
        draws[f].copy_(idx)
    d = draws.cpu().numpy()
    torch.cuda.synchronize()
    ring.close()
    st.close()
    assert all(len(np.unique(r)) == 32 for r in d)
    np.testing.assert_array_equal(d[1234], uniform_draw(2024, 1234 * 32, 32, 1000, 1000, 0))
    counts = np.bincount(d.ravel(), minlength=1000)
    chi2 = ((counts - 128.0) ** 2 / 128.0).sum()
    assert stats.chi2.sf(chi2, 999) > 1e-4, chi2


def test_a_batch_larger_than_the_stored_rollouts_is_refused():
    from distributed_rl_b200 import _lib
    from distributed_rl_b200.replay_server import ServeRing
    st = _store(2, 32, 10)
    ring = ServeRing.create(st, 16, 1)
    try:
        lib = _lib.load()
        launches = lib.b2rl_launch_count()
        with pytest.raises(_lib.B2RLError, match="larger than population"):
            ring.fill_uniform(st, 0, 5, 2)
        assert lib.b2rl_launch_count() == launches          # nothing was launched
        hdr = _take(ring, 0, st.fields)[0]
        torch.cuda.synchronize()
        assert hdr.tolist() == [0, 0]
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


# ---- two processes --------------------------------------------------------------------------------------------------
def _impala_record(rng, T):
    """A rollout as IMPALA/Player.py:176-190 pickles it: [s (T+1, 28224), a (T, 1), mu (T, 1), r (T,), flag]."""
    return [rng.integers(0, 256, (T + 1, 28224), dtype=np.uint8), rng.integers(0, 6, (T, 1)),
            rng.random((T, 1)).astype(np.float32), rng.standard_normal(T).astype(np.float32),
            float(rng.integers(0, 2))]


def _server_main(proxy, cfg_kw, stop, out):
    import time
    from distributed_rl_b200 import impala
    from distributed_rl_b200.replay_server import DeviceReplayServer
    srv = DeviceReplayServer(impala.ImpalaConfig(**cfg_kw), Shim(proxy), slots=3)
    srv.store.seed(4242, 0)
    while not stop.is_set():
        st = srv.serve_once()
        if not (st["ingested"] or st["filled"] or st["released"] or st["updates_applied"]):
            time.sleep(0.0005)
    torch.cuda.synchronize()
    out.put(srv.close(timeout=60))


def test_two_process_impala_round_trip(monkeypatch):
    from distributed_rl_b200 import impala, wire
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200 import replay_server as RS
    N, B, steps, T = 40, 4, 10, 20
    base = dict(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=64, BUFFER_SIZE=16, LEARNER_DEVICE="cuda:0")
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
        recs = [_impala_record(rng, T) for _ in range(N)]
        cols = wire.decode_impala(recs, T)
        conn.rpush("trajectory", *[pickle.dumps(r) for r in recs])
        client = RS.DeviceReplayClient(impala.ImpalaConfig(**base), conn, timeout=180.0)
        served, conv1_frames = [], []
        sample = client.sample

        def rec_sample():
            b = sample()
            if b is not False:
                served.append(([t.clone() for t in b], client.last_idx.clone(), client.last_served,
                               client.last_header.clone(), b[0].data_ptr(), b[0].is_contiguous()))
            return b
        client.sample = rec_sample
        conv1 = R.conv1_fused

        def rec_conv1(frames, rows, *a, **kw):
            conv1_frames.append((frames.data_ptr(), rows))
            return conv1(frames, rows, *a, **kw)
        monkeypatch.setattr(R, "conv1_fused", rec_conv1)
        torch.manual_seed(0)
        L = impala.Learner(impala.ImpalaConfig(**base), connect=conn, start_replay=False, memory=client)
        assert L.memory is client
        assert conn.get(RS.CLIENT_KEY) is not None and conn.get(RS.RING_KEY) is not None
        assert L.run(max_steps=steps) == steps
        torch.cuda.synchronize()
        assert len(served) == steps and client.slots.upd_seq == 0          # no update slot was ever posted
        # conv_1 of every step ran on the served slot's frame table itself: no copy of `state` in between
        assert [p for p, rows in conv1_frames] == [s[4] for s in served] and all(r is None for _, r in conv1_frames)
        seqs = []
        for (s, a, mu, r, d), idx, (k, seq, n), hdr, _, contiguous in served:
            assert contiguous and n == B and hdr.tolist() == [seq, B]
            seqs.append(seq)
            ii = idx.cpu().numpy()
            assert len(set(ii.tolist())) == B and ii.max() < N
            assert s.shape == (T + 1, B, 28224) and a.shape == (T, B) and d.shape == (B,)
            np.testing.assert_array_equal(s.cpu().numpy(), cols[0][ii].transpose(1, 0, 2))
            for got, want in ((a, cols[1]), (mu, cols[2]), (r, cols[3])):
                np.testing.assert_array_equal(got.cpu().numpy(), want[ii].T)
            np.testing.assert_array_equal(d.cpu().numpy(), cols[4][ii])
        assert seqs == sorted(seqs) and len(set(seqs)) == steps
        # the same learner fed the same minibatches through train() ends with the same weights, bit for bit
        torch.manual_seed(0)
        L2 = impala.Learner(impala.ImpalaConfig(**base), connect=None, start_replay=False)
        for b, *_ in served:
            L2.train(b)
        torch.cuda.synchronize()
        for (name, p1), p2 in zip(L.model.state_dict().items(), L2.model.state_dict().values()):
            assert torch.equal(p1, p2), name
        client.close()
        client = None
        stop.set()
        assert out.get(timeout=120)                      # the server saw SERVE_DETACHED before freeing the ring
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
