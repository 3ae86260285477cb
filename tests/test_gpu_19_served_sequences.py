"""GPU tests of the captured R2D2 and IMPALA steps on served minibatches (SERVED_FUSED_STEP) and of R2D2's captured
in-process step (fused_step(use_graph=True)).

One process: a ring created over a local store stands in for the mapped ring; each slot is bound to the learner's
fixed buffers exactly as DeviceReplayClient.acquire binds it (ServeRing.bind), and the bound step (three eager
warm-ups, the capture, then replays after rebinds) is compared, slot by slot and bit for bit, with a learner of the
same weights running train() on a copy of the same slot.  Two processes: a DeviceReplayServer in a `spawn` child
feeds a learner with the flag through run() (the pattern of test_gpu_16 / test_gpu_17)."""
import multiprocessing as mp
import pickle
import time
from types import SimpleNamespace

import numpy as np
import pytest

from shared_redis import RedisManager, Shim

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(autouse=True)
def _deterministic():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    b = torch.backends
    saved = (b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32)
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = True, False, False, False
    yield
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = saved


def _fill(store, n, seed):
    """Hashed frames; valid actions, finite rewards / LSTM states / probabilities, 0/1 done flags."""
    store.fill_hash(n, seed=seed)
    g = torch.Generator(device=store.device).manual_seed(seed)
    names = [f.name for f in store.fields]
    store.field_view("action").random_(0, 6, generator=g)
    store.field_view("reward").normal_(generator=g)
    for name in ("h0", "h1"):
        if name in names:
            store.field_view(name).normal_(0.0, 0.1, generator=g)
    if "notdone" in names:
        store.field_view("notdone").bernoulli_(0.9, generator=g)
    if "mu" in names:
        store.field_view("mu").uniform_(0.1, 1.0, generator=g)
        store.field_view("done").bernoulli_(0.9, generator=g)
    store.build(torch.rand(n, generator=torch.Generator().manual_seed(seed)).to(store.device) + 0.05)


def _local_memory(ring):
    """What the learner's constructor and bound step read from a DeviceReplayClient: the ring's layout, acquire and
    release (driven by the test through _bind)."""
    return SimpleNamespace(ring=ring, acquire=None, release=None, is_alive=lambda: True)


def _bind(ring, k, fields, state):
    ring.bind(ring.slot_ptrs(k)[0][0], fields, state.cur, state.frames, torch.cuda.current_stream())


def _take(ring, k, fields, time_major):
    """A copy of slot k and the client's views of it: header, idx, w, {field: view}."""
    L, B = ring.layout, ring.layout.batch
    buf = torch.empty(L.slot_bytes, dtype=torch.uint8, device="cuda")
    ring.take(k, buf, torch.cuda.current_stream())

    def view(off, nbytes, dtype, shape):
        return buf[off:off + nbytes].view(dtype).view(shape)

    def shape(f):
        return (f.shape[0], B) + tuple(f.shape[1:]) if time_major and f.shape else (B,) + tuple(f.shape)
    out = {f.name: view(L.field_off[i], B * f.nbytes, f.dtype, shape(f)) for i, f in enumerate(fields)}
    return view(0, 16, torch.int64, (2,)), view(L.idx_off, 8 * B, torch.int64, (B,)), \
        view(L.w_off, 4 * B, torch.float32, (B,)), out


def _same_params_and_state(opt_a, opt_b):
    for pa, pb in zip(opt_a.param_groups[0]["params"], opt_b.param_groups[0]["params"]):
        assert torch.equal(pa, pb)
        sa, sb = opt_a.state[pa], opt_b.state[pb]
        assert sa.keys() == sb.keys()
        for key in sa:
            assert torch.equal(sa[key], sb[key]), key


SLOTS = 6          # 3 eager warm-ups, the capture (replayed once), 2 replays after rebinds


def test_r2d2_served_captured_step_equals_train_on_the_slot():
    from distributed_rl_b200 import r2d2, replay as R
    from distributed_rl_b200.replay_server import KINDS, ServeRing
    B, T, N = 8, 80, 40
    fields = R.r2d2_fields(T)
    st = R.DeviceReplay(N, fields, "cuda:0")
    _fill(st, N, 31)
    ring = ServeRing.create(st, B, SLOTS)
    try:
        st.seed(7, 0)
        for k in range(SLOTS):
            ring.fill(st, k, 100 + k, 0.4)
        cfg = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=8, LEARNER_DEVICE="cuda:0")
        torch.manual_seed(0)
        A = r2d2.Learner(r2d2.R2D2Config(**cfg, SERVED_FUSED_STEP=True), start_replay=False,
                         memory=_local_memory(ring))
        torch.manual_seed(0)
        Bl = r2d2.Learner(r2d2.R2D2Config(**cfg), start_replay=False)
        s = A._state()
        for k in range(SLOTS):
            _bind(ring, k, fields, s)
            out = A._bound_step()
            hdr, idx, w, b = _take(ring, k, fields, False)
            info, prio, idx_b = Bl.train(KINDS["r2d2"].batch(b, w, idx))
            torch.cuda.synchronize()
            assert (A._graph is not None) == (k >= A.BOUND_WARMUP), k
            assert hdr.tolist() == [100 + k, B] and s.cur["header"].tolist() == [100 + k, B]
            assert torch.equal(out["idx"], idx_b) and torch.equal(s.cur["w"].view(torch.int32), w.view(torch.int32))
            assert torch.equal(out["prio"], prio), k
            assert torch.equal(out["scalars"][0], info["loss"]) and torch.equal(out["scalars"][1], info["mean_value"])
            assert torch.equal(out["p_norm"], info["p_norm"]), k
            _same_params_and_state(A.optim, Bl.optim)
        assert A.launches_per_step > 0
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


def test_impala_served_captured_step_equals_train_on_the_slot():
    from distributed_rl_b200 import impala, replay as R
    from distributed_rl_b200.replay_server import KINDS, ServeRing
    B, T, N = 16, 20, 48
    fields = R.impala_fields(T)
    st = R.DeviceReplay(N, fields, "cuda:0")
    _fill(st, N, 41)
    ring = ServeRing.create(st, B, SLOTS)
    try:
        st.seed(9, 0)
        for k in range(SLOTS):
            ring.fill_uniform(st, k, 200 + k, T)
        cfg = dict(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=8, LEARNER_DEVICE="cuda:0")
        torch.manual_seed(0)
        A = impala.Learner(impala.ImpalaConfig(**cfg, SERVED_FUSED_STEP=True), start_replay=False,
                           memory=_local_memory(ring))
        torch.manual_seed(0)
        Bl = impala.Learner(impala.ImpalaConfig(**cfg), start_replay=False)
        s = A._bound_state()
        for k in range(SLOTS):
            _bind(ring, k, fields, s)
            out = A._bound_step()
            hdr, idx, w, b = _take(ring, k, fields, True)
            Bl.train(KINDS["impala"].batch(b, w, idx))
            torch.cuda.synchronize()
            assert (A._graph is not None) == (k >= A.BOUND_WARMUP), k
            assert s.cur["header"].tolist() == [200 + k, B] and torch.equal(s.cur["idx"], idx)
            for key in ("vtarget", "advantage", "objActor", "criticLoss"):
                assert torch.equal(out[key], Bl.last[key]), (k, key)
            _same_params_and_state(A.mOptim, Bl.mOptim)
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


def test_r2d2_in_process_captured_step_equals_the_eager_step():
    """fused_step(use_graph=True) draws its own minibatches in the graph: from the same tree, RNG state and weights it
    follows the eager fused_step step for step (its first call is 3 eager warm-ups + the captured step)."""
    from distributed_rl_b200 import r2d2
    B, T, N = 8, 80, 40
    cfg = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0")
    learners = []
    for _ in range(2):
        torch.manual_seed(0)
        L = r2d2.Learner(r2d2.R2D2Config(**cfg), start_replay=False)
        _fill(L.memory.store, N, 51)
        L.memory.store.seed(13, 0)
        learners.append(L)
    G, E = learners
    outs_e = [E.fused_step() for _ in range(4)][-1:]
    outs_g = [{k: v.clone() for k, v in G.fused_step(use_graph=True).items()}]
    assert G._graph is not None and E._graph is None
    for _ in range(3):
        outs_e.append({k: v.clone() for k, v in E.fused_step().items()})
        outs_g.append({k: v.clone() for k, v in G.fused_step(use_graph=True).items()})
    torch.cuda.synchronize()
    for oe, og in zip(outs_e, outs_g):
        for key in ("idx", "prio", "scalars", "p_norm"):
            assert torch.equal(oe[key], og[key]), key
    assert len({tuple(o["idx"].tolist()) for o in outs_g}) > 1          # every replay drew a new minibatch
    assert torch.equal(E.memory.store.priorities(0, N), G.memory.store.priorities(0, N))
    _same_params_and_state(E.optim, G.optim)


# ---- two processes --------------------------------------------------------------------------------------------------
def _server_main(kind, proxy, cfg_kw, stop, out):
    """The replay server process: serve until `stop`, then report the tree's leaves and free the ring."""
    from distributed_rl_b200 import impala, r2d2
    from distributed_rl_b200.replay_server import DeviceReplayServer
    cfg = r2d2.R2D2Config(**cfg_kw) if kind == "r2d2" else impala.ImpalaConfig(**cfg_kw)
    srv = DeviceReplayServer(cfg, Shim(proxy), slots=3)
    srv.store.seed(4242, 0)
    while not stop.is_set():
        st = srv.serve_once()
        if not (st["ingested"] or st["filled"] or st["released"] or st["updates_applied"]):
            time.sleep(0.0005)
    torch.cuda.synchronize()
    leaves = srv.store.priorities(0, srv.cfg.REPLAY_MEMORY_LEN).cpu().numpy()
    out.put((leaves, srv.close(timeout=60)))


def _impala_record(rng, T):
    """A rollout as IMPALA/Player.py:176-190 pickles it: [s (T+1, 28224), a (T, 1), mu (T, 1), r (T,), flag]."""
    return [rng.integers(0, 256, (T + 1, 28224), dtype=np.uint8), rng.integers(0, 6, (T, 1)),
            rng.random((T, 1)).astype(np.float32) + 0.1, rng.standard_normal(T).astype(np.float32),
            float(rng.integers(0, 2))]


@pytest.mark.parametrize("kind", ["r2d2", "impala"])
def test_two_process_served_captured_step(kind):
    from test_wire_cpu import _r2d2_record
    from distributed_rl_b200 import impala, r2d2, wire
    from distributed_rl_b200 import replay_server as RS
    N, B, steps, log_every = 40, 4, 10, 5
    if kind == "r2d2":
        T, mod, Cfg, list_key = 80, r2d2, r2d2.R2D2Config, "experience"
        base = dict(BATCHSIZE=B, FIXED_TRAJECTORY=T, REPLAY_MEMORY_LEN=64, BUFFER_SIZE=16, LEARNER_DEVICE="cuda:0")
    else:
        T, mod, Cfg, list_key = 20, impala, impala.ImpalaConfig, "trajectory"
        base = dict(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=64, BUFFER_SIZE=16, LEARNER_DEVICE="cuda:0")
    ctx = mp.get_context("spawn")
    mgr = RedisManager(ctx=ctx)
    mgr.start()
    child, stop, client = None, ctx.Event(), None
    try:
        proxy = mgr.Redis()
        conn = Shim(proxy)
        out = ctx.Queue()
        child = ctx.Process(target=_server_main, args=(kind, proxy, base, stop, out))
        child.start()
        rng = np.random.default_rng(0)
        if kind == "r2d2":
            recs = [_r2d2_record(rng, T, bool(i % 5 == 0)) for i in range(N)]
            prios = wire.decode_r2d2(recs, T)[1]
        else:
            recs = [_impala_record(rng, T) for _ in range(N)]
            prios = np.ones(N, np.float32)
        conn.rpush(list_key, *[pickle.dumps(r) for r in recs])
        client = RS.DeviceReplayClient(Cfg(**base), conn, timeout=180.0)
        bound, updates, released = [], [], []
        acquire, release, update = client.acquire, client.release, client.update

        def rec_acquire(cur, frames):
            d = acquire(cur, frames)
            if d is not None:
                bound.append(d)
            return d

        def rec_release():
            released.append(client._held)
            release()

        def rec_update(idx, vals):
            updates.append((idx.clone(), vals.clone()))
            update(idx, vals)
        client.acquire, client.release, client.update = rec_acquire, rec_release, rec_update
        torch.manual_seed(0)
        L = mod.Learner(Cfg(**base, SERVED_FUSED_STEP=True), connect=conn, start_replay=False, memory=client)
        n = L.run(max_steps=steps, log_every=log_every) if kind == "r2d2" else L.run(max_steps=steps)
        assert n == steps
        torch.cuda.synchronize()
        assert L._graph is not None                     # steps after the warm-up replayed the captured graph
        assert len(bound) == steps and [d[:2] for d in bound] == released     # every bound slot went back
        seqs = [d[1] for d in bound]
        assert seqs == sorted(seqs) and len(set(seqs)) == steps            # slots were released and refilled
        if kind == "r2d2":
            assert len(updates) == steps - steps // log_every               # the eviction steps skip their write-back
            t0 = time.time()
            while len(client.slots.upd_free) < client.ring.layout.slots or client._pending:
                assert time.time() - t0 < 60, "update slots not handed back"
                client.slots.poll()
                client._flush_updates()
                time.sleep(0.005)
        else:
            assert not updates and client.slots.upd_seq == 0
        want = np.zeros(64, np.float32)
        want[:N] = prios
        for i, v in updates:
            want[i.cpu().numpy()] = v.cpu().numpy()
        client.close()
        client = None
        stop.set()
        leaves, freed = out.get(timeout=120)
        np.testing.assert_array_equal(leaves, want)     # the write-backs reached the server's tree
        assert freed                                    # the server saw SERVE_DETACHED before freeing the ring
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
