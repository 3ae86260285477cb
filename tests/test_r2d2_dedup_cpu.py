"""CPU tests of the frame-deduplicated R2D2 store (R2D2Config.FRAME_DEDUP, DESIGN.md §4.18): the CPU model of strip
records' pool ids over Player-like sequences (a mid-episode sequence adds T / 2 frames), the push geometry, and the
configuration's keys and refusals."""
import importlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from strip_dedup_model import StripDedupModel, max_batch, player_sequences  # noqa: E402


def test_player_sequences_slide_and_follow_the_cut_rule():
    T = 16
    strips, a, r, h0, h1, nd, kind = player_sequences(60, T=T, actors=3, episode=(30, 60), seed=1)
    assert strips.shape == (60, T + 3, 84, 84) and a.shape == (60, T) and h0.shape == (60, 512)
    assert {"first", "mid", "done"} <= set(kind)
    assert (nd[[k == "done" for k in kind]] == 0).all() and (nd[[k == "mid" for k in kind]] == 1).all()
    for s, k in zip(strips, kind):
        if k == "first" and np.array_equal(s[0], s[3]):
            assert np.array_equal(s[0], s[1]) and np.array_equal(s[0], s[2])     # the episode's first stack: o_0 x 4


@pytest.mark.parametrize("T", [16, 80])
def test_a_mid_episode_sequence_adds_half_its_steps(T):
    """Pushed one sequence at a time, in actor-interleaved order: a mid-episode sequence stores exactly T / 2 new
    frames, an episode's first sequence its distinct frames (o_0 once), and a done sequence, which overlaps the one
    before it by less, the frames after that one's last."""
    n = 40 if T == 80 else 120
    strips, *_, kind = player_sequences(n, T=T, actors=4, episode=(3 * T, 6 * T), seed=2)
    m = StripDedupModel(n, 200 * (T + 3), 50 * (T + 3), T)
    for i in range(n):
        m.push(strips[i:i + 1], np.ones(1, np.float32))
    new = np.array(m.new_frames)
    kinds = np.array(kind)
    assert (kinds == "mid").sum() >= n // 3
    assert (new[kinds == "mid"] == T // 2).all()
    for i in np.flatnonzero(kinds == "first"):
        assert new[i] == len({strips[i][j].tobytes() for j in range(T + 3)})
    assert ((new[kinds == "done"] > 0) & (new[kinds == "done"] <= T + 3)).all()
    assert np.array_equal(m.strips(np.arange(n)), strips)


def test_batch_representatives_window_and_eviction():
    """Two equal sequences in one batch share every id (the lower position is stored); a frame older than the
    window is stored again; slots die once F - W frames have been stored since their batch began."""
    T = 8
    R = T + 3
    rng = np.random.default_rng(3)
    x = rng.integers(0, 256, (2, R, 84, 84), dtype=np.uint8)
    m = StripDedupModel(8, 6 * R, R, T)
    m.push(np.stack([x[0], x[0]]), np.ones(2, np.float32))
    assert m.new_frames == [R] and np.array_equal(m.planes[0], m.planes[1])
    m.push(x[1:2], np.ones(1, np.float32))                    # R new frames: x[0]'s are now outside the window
    m.push(x[0:1], np.ones(1, np.float32))
    assert m.new_frames[-1] == R
    assert m.size == 4 and (m.prio[:4] == 1).all()             # 3 R frames since slot 0's batch: F - W = 5 R not yet
    m.push(rng.integers(0, 256, (2, R, 84, 84), dtype=np.uint8), np.ones(2, np.float32))
    assert m.head == 5 * R and m.size == 4                      # slots 0 and 1 (5 R since their batch) died
    assert (m.prio[:2] == 0).all() and (m.prio[2:6] == 1).all()
    # hash collisions (mask 0): every frame keys alike, so inside a batch only copies of its first frame are found;
    # across batches the key table's one entry (the newest frame) is found by the full compare
    c = StripDedupModel(8, 6 * R, 2 * R, T, mask=0)
    c.push(np.stack([x[0], x[1], x[0]]), np.ones(3, np.float32))
    assert c.new_frames == [3 * R - 1] and c.planes[2, 0] == c.planes[0, 0]
    c.push(x[0][::-1].copy()[None], np.ones(1, np.float32))     # its first frame is the newest stored frame
    assert c.new_frames[-1] == R - 1


def test_push_geometry():
    assert max_batch(10_000, 480_000, 16_384, 83) == 65536 // 83 == 789
    assert max_batch(100, 480_000, 16_384, 83) == 100
    assert max_batch(10_000, 5_000, 1_000, 83) == (5_000 - 1_000 - 1) // 83
    assert max_batch(10_000, 100_000, 0, 8) == 8192            # the Ape-X cap is the same scratch


def test_config_geometry_keys_and_refusals(tmp_path, monkeypatch):
    from distributed_rl_b200 import r2d2
    c = r2d2.R2D2Config(FRAME_DEDUP=True, REPLAY_MEMORY_LEN=10_000)
    assert c.FRAME_STRIP                                       # dedup stores strips
    assert r2d2.dedup_geometry(c) == (480_000, 16_384)
    small = r2d2.R2D2Config(FRAME_DEDUP=True, REPLAY_MEMORY_LEN=100, FRAMES_PER_SEQUENCE=41.5)
    with pytest.warns(UserWarning, match="eighth"):
        assert r2d2.dedup_geometry(small) == (4150, 4150 // 8)
    for kw in (dict(HOST_FRAMES=True), dict(PAYLOAD_POOL=64)):
        with pytest.raises(ValueError, match="FRAME_DEDUP"):
            r2d2.R2D2Config(FRAME_DEDUP=True, **kw)
    assert not r2d2.R2D2Config().FRAME_DEDUP and not r2d2.R2D2Config().FRAME_STRIP
    # optional keys of cfg/r2d2.json, through the drop-in configuration module
    cfg = {"ALG": "R2D2", "FIXED_TRAJECTORY": 80, "MEM": 20, "USE_RESCALING": True, "ALPHA": 0.9, "BETA": 0.4,
           "TARGET_FREQUENCY": 2500, "N": 32, "GAMMA": 0.997, "BATCHSIZE": 32, "ACTION_SIZE": 6, "UNROLL_STEP": 5,
           "REPLAY_MEMORY_LEN": 1000, "REDIS_SERVER": "localhost", "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0",
           "BUFFER_SIZE": 100, "optim": {"name": "adam", "lr": 1e-4, "eps": 0.001}, "model": {},
           "FRAME_DEDUP": True, "FRAMES_PER_SEQUENCE": 44, "DEDUP_WINDOW": 4096}
    path = tmp_path / "r2d2.json"
    path.write_text(json.dumps(cfg))
    monkeypatch.setenv("B2RL_CFG", str(path))
    monkeypatch.chdir(tmp_path)
    monkeypatch.syspath_prepend(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dropin"))
    sys.modules.pop("configuration", None)
    try:
        importlib.import_module("configuration")
        got = r2d2.R2D2Config.from_configuration()
    finally:
        sys.modules.pop("configuration", None)
    assert got.FRAME_DEDUP and got.FRAME_STRIP and got.FRAMES_PER_SEQUENCE == 44 and got.DEDUP_WINDOW == 4096
    assert r2d2.dedup_geometry(got) == (44_000, 4096)
    del cfg["FRAME_DEDUP"], cfg["FRAMES_PER_SEQUENCE"], cfg["DEDUP_WINDOW"]
    path.write_text(json.dumps(cfg))
    try:
        importlib.import_module("configuration")
        plain = r2d2.R2D2Config.from_configuration()
    finally:
        sys.modules.pop("configuration", None)
    assert not plain.FRAME_DEDUP and plain.FRAMES_PER_SEQUENCE == r2d2.R2D2Config.FRAMES_PER_SEQUENCE


def test_strip_dedup_fields_and_bindings():
    from distributed_rl_b200 import _lib, replay as R
    f = R.R2D2_DEDUP_FIELDS(80)
    assert f[0].name == "planes" and f[0].nbytes == 4 * 83
    assert [x.name for x in f[1:]] == [x.name for x in R.r2d2_fields(80, strip=True)[1:]]
    per_seq = sum(x.nbytes for x in f)
    assert per_seq == 332 + 4740
    assert dict(_lib.Frames._fields_)["plane_stride"] is _lib.c_i32
    assert _lib.Frames().plane_stride == 0                     # 0 means 8: the Ape-X plane table
