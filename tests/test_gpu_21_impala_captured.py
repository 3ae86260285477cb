"""GPU tests of IMPALA's captured in-process learner step (impala.Learner.fused_step(use_graph=True)) and of its draw,
b2rl_uniform_fetch (csrc/uniform.cu, DeviceReplay.uniform_fetch).

The draw: idx against its numpy restatement (tests/uniform_oracle.py) bit for bit, with the Philox counter advancing
by n; the small fields against a torch gather of the drawn slots, transposed to time-major; the frame rows against
time_major_rows; and the same slots and fields as the served fill (b2rl_serve_fill_uniform) from the same RNG state.
The step: against the same draw followed by the body run eagerly, bit for bit, and against train() on the batch staged
from its idx; replays that follow the ring as ingests move its head and skip slots reserved by an ingest in flight;
and the refusals."""
from types import SimpleNamespace

import numpy as np
import pytest

from test_gpu_17_impala_serve import _store, _take
from test_gpu_19_served_sequences import _fill, _same_params_and_state
from uniform_oracle import uniform_draw

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SMALL = ("action", "mu", "reward", "done")


@pytest.fixture(autouse=True)
def _deterministic():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    b = torch.backends
    saved = (b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32)
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = True, False, False, False
    yield
    b.cudnn.deterministic, b.cudnn.benchmark, b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32 = saved


def _buffers(B, T):
    """uniform_fetch's fixed buffers: idx (B,), action / mu / reward (T, B), done (B,), frame rows ((T+1) * B,)."""
    from distributed_rl_b200 import replay as R
    f = {x.name: x for x in R.impala_fields(T)}
    out = {name: torch.zeros((T, B), dtype=f[name].dtype, device="cuda:0") for name in ("action", "mu", "reward")}
    out.update(done=torch.zeros(B, dtype=f["done"].dtype, device="cuda:0"),
               idx=torch.zeros(B, dtype=torch.int64, device="cuda:0"),
               rows=torch.zeros((T + 1) * B, dtype=torch.int64, device="cuda:0"))
    return out


def _bytes(t):
    return t.contiguous().reshape(-1).view(torch.uint8)


def _time_major_rows(idx, T):
    from distributed_rl_b200.learner_common import time_major_rows
    return time_major_rows(idx, torch.arange(T + 1, device=idx.device).view(T + 1, 1))


@pytest.mark.parametrize("B,T,cap,pushes,evict", [
    (16, 2, 64, 40, 0),          # a partly filled ring; size 40 is not a power of 4, so the cycle walk runs
    (24, 2, 64, 100, 0),         # a full ring that has wrapped: head in mid-ring
    (48, 2, 64, 100, 16),        # size == n: a full permutation of the wrapped valid region
    (200, 20, 256, 300, 20),     # T = 20, several CTAs of draws
])
def test_uniform_fetch_equals_the_oracle_and_the_time_major_gather(B, T, cap, pushes, evict):
    from distributed_rl_b200 import _lib
    st = _store(T, cap, pushes, evict)
    size, _, head = st._sizes()
    assert size == min(cap, pushes) - evict
    out = _buffers(B, T)
    lib = _lib.load()
    try:
        for seed, counter in ((7, 0), (0xFFFF_FFFF_1234, 2 ** 40)):
            st.seed(seed, counter)
            for off in (0, B):                           # a second call draws at counter + B
                n0 = lib.b2rl_launch_count()
                st.uniform_fetch(B, T, out)
                assert lib.b2rl_launch_count() == n0 + 1
                torch.cuda.synchronize()
                idx = out["idx"]
                want = uniform_draw(seed, counter + off, B, size, cap, head)
                np.testing.assert_array_equal(idx.cpu().numpy(), want)
                if B == size:
                    assert sorted(want.tolist()) == sorted(((head - size + np.arange(size)) % cap).tolist())
                for name in SMALL:
                    r = st.field_view(name)[idx]                                # torch gather of the payload
                    r = r.t() if r.dim() == 2 else r                            # (B, T) -> time-major (T, B)
                    assert torch.equal(_bytes(out[name]), _bytes(r)), name
                assert torch.equal(out["rows"], _time_major_rows(idx, T))
    finally:
        torch.cuda.synchronize()
        st.close()


@pytest.mark.parametrize("B", [32, 200])
def test_uniform_fetch_draws_what_the_served_fill_draws(B):
    from distributed_rl_b200.replay_server import ServeRing
    T = 20
    st = _store(T, 256, 300, 20)
    ring = ServeRing.create(st, B, 1)
    try:
        out = _buffers(B, T)
        for seed, counter in ((11, 3), (0xABCD_0123_4567, 2 ** 33 + 5)):
            st.seed(seed, counter)
            st.uniform_fetch(B, T, out)
            st.seed(seed, counter)
            ring.fill_uniform(st, 0, 1, T)
            _, idx, _, got = _take(ring, 0, st.fields)
            torch.cuda.synchronize()
            assert torch.equal(out["idx"], idx)
            for name in SMALL:
                assert torch.equal(_bytes(out[name]), _bytes(got[name])), name
    finally:
        torch.cuda.synchronize()
        ring.close()
        st.close()


def _learner(B, T, N, fill_seed=None, **kw):
    from distributed_rl_b200 import impala
    torch.manual_seed(0)
    L = impala.Learner(impala.ImpalaConfig(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0"),
                       start_replay=False, **kw)
    if fill_seed is not None:
        _fill(L.memory.store, N, fill_seed)
    return L


def _snap(out):
    return {k: v.clone() for k, v in out.items()}


def _eager_step(L):
    """What the captured step replays, run eagerly: the draw into the fixed buffers, then the body."""
    c = L.cfg
    s = L._drawn_state()
    cur = s.cur
    L.memory.store.uniform_fetch(c.BATCHSIZE, c.UNROLL_STEP, cur)
    L._train_core(s.frames, cur["rows"], cur["action"], cur["mu"], cur["reward"], cur["done"], 0)
    return _snap(dict(L.last, idx=cur["idx"]))


KEYS = ("idx", "vtarget", "advantage", "objActor", "criticLoss")


def test_captured_step_equals_the_eager_step_and_train_on_the_staged_batch():
    """From the same weights, replay contents and RNG state, fused_step(use_graph=True) follows the eager draw + body
    step for step (its first call is 3 eager warm-ups + the captured step), each replay on a new minibatch; and a
    replay equals train() on the batch staged from its idx."""
    B, T, N = 16, 20, 48
    E, G = (_learner(B, T, N, fill_seed=61) for _ in range(2))
    for L in (E, G):
        L.memory.store.seed(13, 0)
    outs_e = [_eager_step(E) for _ in range(4)][-1:]
    outs_g = [_snap(G.fused_step(use_graph=True))]
    assert G._graph is not None and G.launches_per_step > 0 and E._graph is None
    torch.cuda.synchronize()
    _same_params_and_state(E.mOptim, G.mOptim)
    for _ in range(3):
        outs_e.append(_eager_step(E))
        outs_g.append(_snap(G.fused_step(use_graph=True)))
        torch.cuda.synchronize()
        _same_params_and_state(E.mOptim, G.mOptim)
    for oe, og in zip(outs_e, outs_g):
        for key in KEYS:
            assert torch.equal(oe[key], og[key]), key
    assert len({tuple(o["idx"].tolist()) for o in outs_g}) == len(outs_g)     # every replay drew a new minibatch
    # one more replay, against train() on the batch staged from its idx as Replay.bufferSave stages it
    og = _snap(G.fused_step(use_graph=True))
    b = E.memory.store.gather(og["idx"])
    E.train((b["state"].transpose(0, 1).contiguous(), b["action"].t().contiguous(), b["mu"].t().contiguous(),
             b["reward"].t().contiguous(), b["done"]))
    torch.cuda.synchronize()
    for key in KEYS[1:]:
        assert torch.equal(og[key], E.last[key]), key
    _same_params_and_state(E.mOptim, G.mOptim)


def _rollouts(rng, k, T):
    """k valid rollouts as host arrays: frames, actions in [0, 6), behaviour probabilities, rewards, done flags."""
    return [rng.integers(0, 256, size=(k, T + 1, 28224), dtype=np.uint8), rng.integers(0, 6, size=(k, T)).astype(np.int32),
            rng.uniform(0.05, 0.9, size=(k, T)).astype(np.float32), rng.standard_normal((k, T)).astype(np.float32),
            (rng.random(k) > 0.3).astype(np.float32)]


def test_captured_step_follows_the_ring_and_skips_slots_reserved_by_an_ingest_in_flight():
    """Replays draw from the valid region [head - size, head) as it is at each call: after pushes that wrap the head,
    with a push_begin in flight (its reserved slots are never drawn) and after its push_commit (they are)."""
    B, T, N, seed = 8, 2, 16, 5
    L = _learner(B, T, N)
    mem, st = L.memory, L.memory.store
    rng = np.random.default_rng(3)
    mem.push_arrays(*_rollouts(rng, 12, T))
    st.seed(seed, 0)
    counter = [3 * B]                                   # the first call's captured draw follows its 3 warm-ups'

    def replay():
        out = L.fused_step(use_graph=True)
        size, cap, head = st._sizes()
        idx = out["idx"].cpu().numpy()
        np.testing.assert_array_equal(idx, uniform_draw(seed, counter[0], B, size, cap, head))
        counter[0] += B
        return set(idx.tolist())

    replay()
    assert L._graph is not None
    for k in (5, 6):                                    # head 12 -> 1 -> 7: the ring is full and wraps twice
        mem.push_arrays(*_rollouts(rng, k, T))
        replay()
    assert st._sizes() == (16, 16, 7)
    cols = [torch.from_numpy(x).pin_memory() for x in _rollouts(rng, 8, T)]
    st.push_begin(cols, 8)                              # slots 7..14 reserved, their copy in flight
    reserved = set(range(7, 15))
    assert st._sizes() == (8, 16, 7)
    for _ in range(2):                                  # 8 of the 8 kept rollouts: 15, 0..6
        assert replay() == set(range(16)) - reserved
    st.push_commit(torch.ones(8))
    assert st._sizes() == (16, 16, 15)
    drawn = replay() | replay()
    assert drawn & reserved


def test_refusals():
    """n > size: ValueError from DeviceReplay.uniform_fetch and from the captured step, an error from the library,
    and nothing launched.  A store whose fields are not a time-major rollout is refused.  A served memory is refused."""
    from distributed_rl_b200 import _lib, replay as R
    lib = _lib.load()
    st = _store(2, 32, 10)
    out = _buffers(16, 2)
    try:
        n0 = lib.b2rl_launch_count()
        with pytest.raises(ValueError, match="larger than population"):
            st.uniform_fetch(16, 2, out)
        with pytest.raises(_lib.B2RLError, match="larger than population"):
            _lib.check(lib.b2rl_uniform_fetch(st._h, 16, 2, out["idx"].data_ptr(), None, None, None))
        assert lib.b2rl_launch_count() == n0
    finally:
        st.close()
    seq = R.DeviceReplay(4, R.r2d2_fields(80), "cuda:0")       # action / reward: 80 words, not a T = 20 rollout's
    try:
        seq.fill_hash(4)
        n0 = lib.b2rl_launch_count()
        with pytest.raises(_lib.B2RLError, match="time-major rollout"):
            _lib.check(lib.b2rl_uniform_fetch(seq._h, 2, 20, out["idx"].data_ptr(), None, None, None))
        assert lib.b2rl_launch_count() == n0
    finally:
        torch.cuda.synchronize()
        seq.close()
    L = _learner(16, 2, 32)
    L.memory.push_arrays(*_rollouts(np.random.default_rng(0), 10, 2))
    n0 = lib.b2rl_launch_count()
    with pytest.raises(ValueError, match="larger than population"):
        L.fused_step(use_graph=True)
    assert lib.b2rl_launch_count() == n0 and L._graph is None
    S = _learner(16, 2, 32, memory=SimpleNamespace(is_alive=lambda: True))
    with pytest.raises(RuntimeError, match="served replay"):
        S.fused_step(use_graph=True)
