"""CPU checks of the frame-deduplicated Ape-X store's rule (tests/dedup_model.py): pool ids, the window, both
eviction conditions, and what the reference actor's records deduplicate to."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dedup_model import DedupModel, frame_keys, max_batch, player_records  # noqa: E402


def _check_live_stacks(m, s, ns, order):
    """Every live slot's pool ids name exactly the stacks pushed into it (order[i]: record of push position i)."""
    live = m.live_slots()
    got_s, got_ns = m.stacks(live)
    # slot -> last record pushed into it
    n = len(order)
    last = {}
    for i in range(n):
        last[i % m.cap] = order[i]
    rec = np.array([last[int(sl)] for sl in live])
    assert np.array_equal(got_s, s[rec]) and np.array_equal(got_ns, ns[rec])


def test_player_stream_stores_about_three_frames_per_record():
    s, ns, a, r, d = player_records(2000, actors=8, seed=1)
    m = DedupModel(capacity=4096, pool_frames=4 * 4096, window=1024)
    m.push(s, ns, np.ones(len(a), np.float32))
    per_record = m.head / len(a)
    # one new frame per env step, plus the repeated first frame at an episode start: ~1 frame per record once s'
    # (3 steps ahead) has been seen, 4 at the first records of an episode
    assert per_record < 3.0, per_record
    assert m.size == len(a)
    _check_live_stacks(m, s, ns, np.arange(len(a)))


def test_episode_start_is_one_frame():
    s, ns, a, r, d = player_records(1, actors=1, seed=2)
    m = DedupModel(capacity=8, pool_frames=64, window=16)
    m.push(s, ns, np.ones(1, np.float32))
    # s = f0 f0 f0 f0, s' = f0 f1 f2 f3: four distinct frames
    assert m.head == 4
    assert (m.planes[0, :4] == m.planes[0, 0]).all()


def test_no_repeats_stores_every_frame_and_evicts_by_frames():
    rng = np.random.default_rng(3)
    n, cap, F, W = 60, 64, 160, 16
    s = rng.integers(0, 256, (n, 4, 84, 84), dtype=np.uint8)
    ns = rng.integers(0, 256, (n, 4, 84, 84), dtype=np.uint8)
    m = DedupModel(cap, F, W)
    for i in range(0, n, 6):
        m.push(s[i:i + 6], ns[i:i + 6], np.full(len(s[i:i + 6]), 1.0, np.float32))
    assert m.head == 8 * n
    # a slot is live while fewer than F - W = 144 frames (18 records of 8 new frames) were stored since its batch began
    assert m.size <= (F - W) // 8 + 6 and m.size >= (F - W) // 8 - 6
    for slot in m.live_slots():
        assert m.head - m.ins[slot] < F - W
    dead = np.setdiff1d(np.arange(n) % cap, m.live_slots())
    assert (m.prio[dead] == 0).all()
    _check_live_stacks(m, s, ns, np.arange(n))


def test_slot_ring_wrap_is_the_other_eviction():
    s, ns, a, r, d = player_records(300, actors=8, seed=4)
    m = DedupModel(capacity=64, pool_frames=4 * 64 * 4, window=32)
    for i in range(0, 300, 10):
        m.push(s[i:i + 10], ns[i:i + 10], np.ones(10, np.float32))
    assert m.size == 64       # the slot ring, not the frame rule, bounds it: ~1-3 frames per record
    _check_live_stacks(m, s, ns, np.arange(300))


def test_repeats_outside_the_window_are_stored_again():
    rng = np.random.default_rng(5)
    f = rng.integers(0, 256, (84, 84), dtype=np.uint8)
    other = rng.integers(0, 256, (40, 84, 84), dtype=np.uint8)
    m = DedupModel(capacity=64, pool_frames=512, window=16)
    st = np.broadcast_to(f, (1, 4, 84, 84)).copy()
    m.push(st, st, np.ones(1, np.float32))
    assert m.head == 1
    m.push(st, st, np.ones(1, np.float32))     # inside the window: reused
    assert m.head == 1
    for i in range(0, 40, 4):                   # 40 distinct frames: f falls out of the 16-frame window
        m.push(other[None, i:i + 4], other[None, i:i + 4], np.ones(1, np.float32))
    assert m.head == 41
    m.push(st, st, np.ones(1, np.float32))
    assert m.head == 42
    assert np.array_equal(m.stacks([m.slot_head - 1])[0][0], st[0])


def test_identical_frames_in_a_batch_take_the_lowest_position():
    rng = np.random.default_rng(6)
    f = rng.integers(0, 256, (3, 84, 84), dtype=np.uint8)
    s = f[[0, 1, 0, 1]][None].repeat(2, 0)
    ns = f[[2, 2, 0, 1]][None].repeat(2, 0)
    m = DedupModel(capacity=8, pool_frames=64, window=8)
    m.push(s, ns, np.ones(2, np.float32))
    assert m.head == 3
    assert m.planes[0].tolist() == [0, 1, 0, 1, 2, 2, 0, 1] and m.planes[1].tolist() == m.planes[0].tolist()


def test_forced_collisions_only_cost_copies():
    s, ns, a, r, d = player_records(200, actors=8, seed=7)
    exact = DedupModel(256, 1024, 128)
    coll = DedupModel(256, 1024, 128, mask=0)
    for m in (exact, coll):
        m.push(s, ns, np.ones(200, np.float32))
        _check_live_stacks(m, s, ns, np.arange(200))
    assert coll.head >= exact.head
    assert (frame_keys(s[:3].reshape(-1, 84, 84), 0) == 0).all()


def test_frame_key_is_content_only():
    rng = np.random.default_rng(8)
    x = rng.integers(0, 256, (5, 84, 84), dtype=np.uint8)
    k = frame_keys(x)
    assert len(set(k.tolist())) == 5 and (k < np.uint64(1 << 63)).all()
    assert (frame_keys(x.copy()) == k).all()
    y = x.copy()
    y[2, 83, 83] ^= 1
    assert frame_keys(y)[2] != k[2]


def test_large_pushes_are_split_into_max_batch_chunks():
    assert max_batch(1 << 21, 4 << 21, 1 << 20) == 8192
    assert max_batch(64, 160, 16) == 17
    s, ns, a, r, d = player_records(100, seed=9)
    one, parts = DedupModel(128, 160, 16), DedupModel(128, 160, 16)
    one.push(s, ns, np.ones(100, np.float32))
    for i in range(0, 100, 17):
        parts.push(s[i:i + 17], ns[i:i + 17], np.ones(len(s[i:i + 17]), np.float32))
    assert one.head == parts.head and np.array_equal(one.planes, parts.planes) and one.size == parts.size


def test_config_geometry_and_defaults():
    from distributed_rl_b200.apex import ApexConfig, dedup_geometry
    c = ApexConfig()
    assert c.FRAME_DEDUP is False and c.FRAMES_PER_TRANSITION == 4.0 and c.DEDUP_WINDOW == 1 << 20
    assert dedup_geometry(ApexConfig(REPLAY_MEMORY_LEN=1 << 21)) == (4 << 21, 1 << 20)
    assert dedup_geometry(ApexConfig(REPLAY_MEMORY_LEN=1000, FRAMES_PER_TRANSITION=3.5, DEDUP_WINDOW=400)) == (3500, 400)


def test_configuration_reads_the_dedup_keys(tmp_path, monkeypatch):
    import importlib
    import json
    cfg = tmp_path / "ape_x.json"
    keys = dict(ALPHA=0.6, BETA=0.4, TARGET_FREQUENCY=2500, N=1, GAMMA=0.99, BATCHSIZE=32, ACTION_SIZE=6,
                UNROLL_STEP=3, REPLAY_MEMORY_LEN=1000, REDIS_SERVER="localhost", DEVICE="cpu", LEARNER_DEVICE="cpu",
                BUFFER_SIZE=100, optim={}, model={})
    cfg.write_text(json.dumps({"ALG": "APE_X", "FRAME_DEDUP": True, "DEDUP_WINDOW": 4096, **keys}))
    monkeypatch.setenv("B2RL_CFG", str(cfg))
    monkeypatch.chdir(tmp_path)
    dropin = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dropin")
    monkeypatch.syspath_prepend(dropin)
    sys.modules.pop("configuration", None)
    try:
        C = importlib.import_module("configuration")
        assert C.FRAME_DEDUP is True and C.DEDUP_WINDOW == 4096 and not hasattr(C, "FRAMES_PER_TRANSITION")
    finally:
        sys.modules.pop("configuration", None)



def test_a_capped_window_warns():
    from distributed_rl_b200.apex import ApexConfig, dedup_geometry
    with pytest.warns(UserWarning, match="DEDUP_WINDOW"):
        assert dedup_geometry(ApexConfig(REPLAY_MEMORY_LEN=1000)) == (4000, 500)
