"""CPU tests of the frame-deduplicated IMPALA store (ImpalaConfig.FRAME_DEDUP, DESIGN.md §4.20): the strip model of
tests/strip_dedup_model.py, unchanged, at R = 4 (T + 1) (tests/impala_rollouts.py) over Player-like rollouts (a
mid-episode rollout adds T frames, a padded one only its own steps), chunked pushes against one rollout at a time, the push geometry, and the configuration's keys,
geometry warning and refusals."""
import importlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from impala_rollouts import player_rollouts, rollout_frames as _frames, rollout_model  # noqa: E402
from strip_dedup_model import max_batch  # noqa: E402


def test_player_rollouts_slide_and_follow_the_cut_and_pad_rule():
    T = 6
    state, a, mu, r, done, kind = player_rollouts(120, T=T, actors=3, episode=(10, 30), p_done=0.15, seed=1)
    assert state.shape == (120, T + 1, 28224) and a.shape == mu.shape == r.shape == (120, T) and done.shape == (120,)
    assert {"first", "mid", "padded"} <= set(kind)
    kinds = np.array(kind)
    assert (done[kinds == "padded"] == 0).all() and (done[kinds == "mid"] == 1).any()   # a full rollout may end a life
    st = state.reshape(120, T + 1, 4, 84, 84)
    for s, k in zip(st, kind):
        if k == "mid":             # stack t + 1 is stack t shifted by one frame
            assert all(np.array_equal(s[t + 1, :3], s[t, 1:]) for t in range(T))
        if k == "first" and np.array_equal(s[0, 0], s[0, 3]):
            assert np.array_equal(s[0, 0], s[0, 1]) and np.array_equal(s[0, 0], s[0, 2])   # o_0 four times


@pytest.mark.parametrize("T", [4, 20])
def test_new_frames_per_rollout(T):
    """Pushed one rollout at a time in actor-interleaved order, with a window that reaches back past every actor's
    previous rollout: a mid-episode rollout stores exactly T new frames (its first stack is the previous rollout's
    bootstrap stack), a padded one at most T (the padding is the previous rollout's), an episode's first at most
    T + 1 (o_0 once); and the pool ids name every pushed frame."""
    n = 160 if T == 4 else 60
    state, *_, kind = player_rollouts(n, T=T, actors=4, episode=(3 * T, 8 * T), p_done=0.2 / T, seed=2)
    R = 4 * (T + 1)
    m = rollout_model(n, 4 * n * R, n * R, T)
    for i in range(n):
        m.push(_frames(state[i:i + 1]), np.ones(1, np.float32))
    new = np.array(m.new_frames)
    kinds = np.array(kind)
    assert (kinds == "mid").sum() >= n // 3 and (kinds == "padded").sum() >= 1
    assert (new[kinds == "mid"] == T).all()
    assert ((new[kinds == "padded"] >= 1) & (new[kinds == "padded"] <= T)).all()
    assert (new[kinds == "first"] <= T + 1).all()
    assert new.mean() < T + 1
    assert np.array_equal(m.strips(np.arange(n)).reshape(state.shape), state)


def test_a_chunked_push_stores_what_one_rollout_at_a_time_stores():
    """Inside a batch a frame reuses the lowest position holding it, which is the frame one-at-a-time pushes would
    have stored first; misses take their sequence numbers in batch order.  So while the window covers every reuse,
    pushes of max_batch chunks give the same pool ids, pool and head as pushes of one rollout."""
    T, n = 4, 200
    R = 4 * (T + 1)
    state, *_ = player_rollouts(n, T=T, actors=6, episode=(10, 40), p_done=0.1, seed=5)
    F, W = 6 * n * R, 2 * n * R
    one, chunked = rollout_model(64, F, W, T), rollout_model(64, F, W, T)    # max_batch 64
    for i in range(n):
        one.push(_frames(state[i:i + 1]), np.ones(1, np.float32))
    chunked.push(_frames(state), np.ones(n, np.float32))
    assert len(chunked.new_frames) == -(-n // max_batch(64, F, W, R)) == 4
    assert chunked.head == one.head < 0.4 * n * R
    assert np.array_equal(chunked.planes, one.planes) and np.array_equal(chunked.pool, one.pool)


def test_window_expiry_and_liveness_on_rollouts():
    """A frame older than the window is stored again; a slot dies once F - W frames have been stored since its batch
    began, oldest first, so the live slots stay the contiguous region [head - size, head) of the ring."""
    T, cap = 4, 64
    R = 4 * (T + 1)
    state, *_ = player_rollouts(300, T=T, actors=5, episode=(10, 40), p_done=0.1, seed=7)
    F, W = 10 * R, 2 * R                                        # F - W frames: fewer than 64 rollouts' new ones
    m = rollout_model(cap, F, W, T)
    pushed = 0
    for a in range(0, 300, 7):
        chunk = state[a:a + 7]
        m.push(_frames(chunk), np.ones(len(chunk), np.float32))
        pushed += len(chunk)
        live = m.live_slots()
        assert (m.prio[live] == 1).all() and (np.delete(m.prio, live) == 0).all()
        # the live slots hold the last `size` rollouts pushed, their frames intact in the pool
        assert np.array_equal(m.strips(live).reshape(-1, T + 1, 28224), state[pushed - m.size:pushed])
    assert m.head > F and 0 < m.size < cap                      # the pool wrapped and killed slots
    # a rollout whose frames have all left the window is stored again in full
    x = _frames(state[:1])
    before = m.head
    m.push(x, np.ones(1, np.float32))
    assert m.head - before == len({f.tobytes() for f in x[0]})


def test_push_geometry():
    assert max_batch(10_000, 240_000, 16_384, 84) == 65536 // 84 == 780
    assert max_batch(500, 240_000, 16_384, 84) == 500
    assert max_batch(10_000, 2_400, 300, 84) == (2_400 - 300 - 1) // 84


def test_config_geometry_keys_and_refusals(tmp_path, monkeypatch):
    from distributed_rl_b200 import impala, replay as R
    assert not impala.ImpalaConfig().FRAME_DEDUP
    c = impala.ImpalaConfig(FRAME_DEDUP=True, REPLAY_MEMORY_LEN=10_000)
    assert impala.dedup_geometry(c) == (240_000, 16_384)
    small = impala.ImpalaConfig(FRAME_DEDUP=True, REPLAY_MEMORY_LEN=100, FRAMES_PER_ROLLOUT=22.5)
    with pytest.warns(UserWarning, match="eighth"):
        assert impala.dedup_geometry(small) == (2250, 2250 // 8)
    # the store's refusals need no device: they are raised before the handle is touched
    for call, exc, msg in ((lambda: R.RolloutDedupReplay.push_begin(None, [None], 4), ValueError, "pipelined"),
                           (lambda: R.RolloutDedupReplay.ingest_pipelined(None, None), ValueError, "pipelined"),
                           (lambda: R.RolloutDedupReplay.fill_hash(None, 4), ValueError, "hashable"),
                           (lambda: R.RolloutDedupReplay.frame_source(None, "next_state"), KeyError, "next_state")):
        with pytest.raises(exc, match=msg):
            call()
    # optional keys of cfg/impala.json, through the drop-in configuration module
    cfg = {"ALG": "IMPALA", "C_LAMBDA": 1.0, "C_VALUE": 1.0, "P_VALUE": 1.0, "ENTROPY_R": 0.01, "GAMMA": 0.99,
           "BATCHSIZE": 32, "ACTION_SIZE": 6, "UNROLL_STEP": 20, "REPLAY_MEMORY_LEN": 1000,
           "REDIS_SERVER": "localhost", "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0", "BUFFER_SIZE": 100,
           "optim": {"name": "rmsprop", "lr": 6e-4, "decay": 0}, "model": {},
           "FRAME_DEDUP": True, "FRAMES_PER_ROLLOUT": 26, "DEDUP_WINDOW": 2048}
    path = tmp_path / "impala.json"
    path.write_text(json.dumps(cfg))
    monkeypatch.setenv("B2RL_CFG", str(path))
    monkeypatch.chdir(tmp_path)
    monkeypatch.syspath_prepend(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dropin"))
    sys.modules.pop("configuration", None)
    try:
        importlib.import_module("configuration")
        got = impala.ImpalaConfig.from_configuration()
    finally:
        sys.modules.pop("configuration", None)
    assert got.FRAME_DEDUP and got.FRAMES_PER_ROLLOUT == 26 and got.DEDUP_WINDOW == 2048
    assert impala.dedup_geometry(got) == (26_000, 2048)
    del cfg["FRAME_DEDUP"], cfg["FRAMES_PER_ROLLOUT"], cfg["DEDUP_WINDOW"]
    path.write_text(json.dumps(cfg))
    try:
        importlib.import_module("configuration")
        plain = impala.ImpalaConfig.from_configuration()
    finally:
        sys.modules.pop("configuration", None)
    assert not plain.FRAME_DEDUP and plain.FRAMES_PER_ROLLOUT == impala.ImpalaConfig.FRAMES_PER_ROLLOUT


def test_rollout_dedup_fields_and_bindings():
    from distributed_rl_b200 import _lib, replay as R
    f = R.IMPALA_DEDUP_FIELDS(20)
    assert f[0].name == "planes" and f[0].nbytes == 4 * 84
    assert [x.name for x in f[1:]] == [x.name for x in R.impala_fields(20)[1:]]
    small = sum(x.nbytes for x in f[1:])
    assert small == 244
    assert 24 * 7056 + f[0].nbytes + small == 169_924               # bytes per slot at the default pool
    assert sum(x.nbytes for x in R.impala_fields(20)) == 592_948     # a stack store's slot
    assert "b2rl_dedup_attach_rollouts" in _lib.SIGNATURES
