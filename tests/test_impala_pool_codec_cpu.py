"""CPU tests of the coded IMPALA frame pool (ImpalaConfig.STAGED_POOL_CODEC, R.RolloutDedupReplay(pool_bytes=...),
DESIGN.md §4.23): the synthetic Atari-like rollouts; the staging map of b2rl_dedup_stage_rollouts (first occurrence,
padded rollouts, a rollout of one id); the store's model, the unit-ring strip model at R = 4 (T + 1), against the
frame-only rollout model and with the byte rule binding past several wraps; the configuration keys, defaults and
refusals; and the refusals of the new entry points before any CUDA work."""
import importlib
import json
import os
import sys
import types

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pool_codec_model as M                                   # noqa: E402
from impala_atari_rollouts import atari_rollouts, staging_map  # noqa: E402
from impala_rollouts import rollout_frames, rollout_model      # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from distributed_rl_b200 import build, _lib
    build.build()
    return _lib.load()


def test_atari_rollouts_are_player_like():
    T = 6
    state, a, mu, r, done, kind = atari_rollouts(60, T=T, actors=3, episode=(20, 40), p_done=0.05, seed=1)
    assert state.shape == (60, T + 1, 28224) and state.dtype == np.uint8 and a.shape == mu.shape == (60, T)
    frames = rollout_frames(state)
    assert np.array_equal(frames[0, 0], frames[0, 3])            # an episode starts with its first frame four times
    assert np.array_equal(frames[0, 4:7], frames[0, 1:4])        # stack t + 1 repeats three frames of stack t
    assert any(np.array_equal(state[j, 0], state[0, T]) for j in range(1, 60))   # the bootstrap stack starts the
                                                                                # actor's next rollout
    assert {"first", "mid", "padded"} <= set(kind)
    enc = [M.units(f) for f in frames[:4].reshape(-1, 84, 84)]
    assert max(enc) < M.RAW_UNITS // 8                           # compressible, unlike impala_rollouts' random frames


def test_staging_map_is_the_first_occurrence_of_each_id():
    T = 20
    R = 4 * (T + 1)
    F = 5000
    state, *_ , kind = atari_rollouts(40, T=T, actors=4, seed=2)
    m = rollout_model(64, F, 600, T)
    m.push(rollout_frames(state), np.ones(40, np.float32))
    planes = m.planes[:40]
    staged = staging_map(planes, F)
    assert staged.shape == (40, R) and staged.dtype == np.int32
    for k in range(40):
        row = staged[k] - k * R
        assert (row <= np.arange(R)).all() and (planes[k][row] == planes[k]).all()
        firsts = np.unique(row)
        assert len(firsts) == len(np.unique(planes[k]))             # one staged frame per distinct id
        assert (row[firsts] == firsts).all()                        # a first occurrence maps to itself
        # the staged pool holds frame i of the rollout at k R + i for every first occurrence i: reading row k through
        # the staged plane table gives the rollout's frames
        pool = {k * R + i: rollout_frames(state)[k, i] for i in firsts}
        assert all(np.array_equal(pool[staged[k, c]], rollout_frames(state)[k, c]) for c in range(R))
    full = [k for k in range(40) if kind[k] != "padded"]
    distinct = [len(np.unique(planes[k])) for k in full]
    assert 4 * (T + 1) // 4 <= np.mean(distinct) <= T + 4            # about 21 of the 84 frames of a full rollout
    padded = [k for k in range(40) if kind[k] == "padded"]
    assert padded and all(len(np.unique(planes[k])) <= T + 4 for k in padded)


def test_staging_map_of_one_id_and_of_ids_outside_the_pool():
    R, F = 84, 1000
    same = np.full((3, R), 7, np.int32)
    assert np.array_equal(staging_map(same, F), np.repeat(np.arange(3)[:, None] * R, R, axis=1))
    odd = np.array([[5, 1005, -1, 2 ** 31 - 1, 5] + [0] * (R - 5)], np.int32)
    s = staging_map(odd, F)[0]
    # ids are taken mod F as unsigned: 1005 names entry 5, and -1 (2^32 - 1) entry 295, as 2^31 - 1 names 647
    assert s[:5].tolist() == [0, 0, 2, 3, 0] and (2 ** 32 - 1) % F == 295 and (2 ** 31 - 1) % F == 647
    assert (s[5:] == 5).all()


def test_unit_ring_model_with_a_large_ring_gives_the_rollout_models_ids():
    T, cap, F, W = 4, 48, 400, 40
    R = 4 * (T + 1)
    state, *_ = atari_rollouts(160, T=T, actors=4, episode=(20, 40), seed=3)
    frames = rollout_frames(state)
    prio = np.linspace(0.1, 2.0, 160).astype(np.float32)
    a, b = rollout_model(cap, F, W, T), M.CodedStripDedupModel(cap, F, W, 4 * T + 1, (F + 1) * M.RAW_UNITS)
    assert b.R == R
    for i in range(0, 160, 7):
        a.push(frames[i:i + 7], prio[i:i + 7])
        b.push(frames[i:i + 7], prio[i:i + 7])
        np.testing.assert_array_equal(a.planes, b.planes)
        np.testing.assert_array_equal(a.prio, b.prio)
        assert a.head == b.head
    assert b.head > F and 0 < b.units < b.P
    live = b.live_slots()
    np.testing.assert_array_equal(b.strips(live), a.strips(live))
    np.testing.assert_array_equal(b.strips(live), frames[160 - len(live):])


def test_unit_ring_model_with_the_byte_rule_binding_past_several_wraps():
    T, cap, F, W = 4, 128, 6000, 24
    R = 4 * (T + 1)
    state, *_ = atari_rollouts(400, T=T, actors=4, episode=(20, 40), seed=4)
    frames = rollout_frames(state)
    frames[::3, 5] = np.random.default_rng(5).integers(0, 256, frames[::3, 5].shape, dtype=np.uint8)   # raw frames
    P = (W + 2 + 2 * R) * M.RAW_UNITS + 21 * 16                    # the window and two rollouts of raw frames
    m, plain = M.CodedStripDedupModel(cap, F, W, 4 * T + 1, P), rollout_model(cap, F, W, T)
    assert M.coded_max_batch(cap, F, W, R, P) == 2
    prio = np.ones(400, np.float32)
    for i in range(0, 400, 2):
        m.push(frames[i:i + 2], prio[i:i + 2])
        plain.push(frames[i:i + 2], prio[i:i + 2])
        np.testing.assert_array_equal(m.planes, plain.planes)      # ids are the frame rule's
        live = m.live_slots()
        if i % 40 == 0 or i == 398:                                # no live slot names an overwritten frame
            np.testing.assert_array_equal(m.strips(live), frames[i + 2 - len(live):i + 2])
        ent = np.unique(m.planes[live])
        assert ((m.foff[ent] % P) + m.flen[ent] <= P).all()        # nothing straddles the ring's end
        assert (m.units - m.uins[live] < P - (W + 1) * M.RAW_UNITS).all()
    assert m.units > 3 * P
    assert len(m.live_slots()) < len(plain.live_slots())           # the byte rule binds before the frame rule


def _configuration(tmp_path, monkeypatch, **extra):
    from distributed_rl_b200 import impala
    cfg = {"ALG": "IMPALA", "C_LAMBDA": 1.0, "C_VALUE": 1.0, "P_VALUE": 1.0, "ENTROPY_R": 0.01, "GAMMA": 0.99,
           "BATCHSIZE": 32, "ACTION_SIZE": 6, "UNROLL_STEP": 20, "REPLAY_MEMORY_LEN": 1000,
           "REDIS_SERVER": "localhost", "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0", "BUFFER_SIZE": 100,
           "optim": {"name": "rmsprop", "lr": 6e-4, "decay": 0}, "model": {}, **extra}
    path = tmp_path / "impala.json"
    path.write_text(json.dumps(cfg))
    monkeypatch.setenv("B2RL_CFG", str(path))
    monkeypatch.chdir(tmp_path)
    monkeypatch.syspath_prepend(os.path.join(REPO, "dropin"))
    sys.modules.pop("configuration", None)
    try:
        importlib.import_module("configuration")
        return impala.ImpalaConfig.from_configuration()
    finally:
        sys.modules.pop("configuration", None)


def test_pool_codec_keys_defaults_and_refusals(tmp_path, monkeypatch):
    from distributed_rl_b200 import impala
    assert impala.ImpalaConfig.STAGED_POOL_CODEC is False and impala.ImpalaConfig.POOL_BYTES_PER_ROLLOUT is None
    c = impala.ImpalaConfig(FRAME_DEDUP=True, STAGED_POOL_CODEC=True, REPLAY_MEMORY_LEN=10_000)
    F, W = impala.dedup_geometry(c)
    assert (F, W) == (240_000, 16_384) and impala.pool_bytes(c) == (F + 1) * 7072
    assert impala.pool_bytes(impala.ImpalaConfig(FRAME_DEDUP=True)) is None
    c2 = impala.ImpalaConfig(FRAME_DEDUP=True, STAGED_POOL_CODEC=True, REPLAY_MEMORY_LEN=1000,
                             POOL_BYTES_PER_ROLLOUT=7300.7)
    assert impala.pool_bytes(c2) == 7_300_700 // 16 * 16
    with pytest.raises(ValueError, match="STAGED_POOL_CODEC.*FRAME_DEDUP"):
        impala.ImpalaConfig(STAGED_POOL_CODEC=True)
    with pytest.raises(ValueError, match="POOL_BYTES_PER_ROLLOUT"):
        impala.ImpalaConfig(FRAME_DEDUP=True, POOL_BYTES_PER_ROLLOUT=8000.0)
    with pytest.raises(ValueError, match="POOL_BYTES_PER_ROLLOUT"):
        impala.ImpalaConfig(FRAME_DEDUP=True, STAGED_POOL_CODEC=True, POOL_BYTES_PER_ROLLOUT=0)
    got = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True, STAGED_POOL_CODEC=True, POOL_BYTES_PER_ROLLOUT=9000)
    assert got.FRAME_DEDUP and got.STAGED_POOL_CODEC and got.POOL_BYTES_PER_ROLLOUT == 9000
    assert impala.pool_bytes(got) == 9_000_000
    plain = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True)
    assert not plain.STAGED_POOL_CODEC and plain.POOL_BYTES_PER_ROLLOUT is None
    with pytest.raises(ValueError, match="STAGED_POOL_CODEC"):
        _configuration(tmp_path, monkeypatch, STAGED_POOL_CODEC=True)


def test_entry_points_refuse_bad_arguments_before_any_cuda_work(lib):
    from distributed_rl_b200 import _lib
    assert "b2rl_dedup_attach_rollouts_coded" in _lib.SIGNATURES and "b2rl_dedup_stage_rollouts" in _lib.SIGNATURES
    launches = lib.b2rl_launch_count()
    M64 = 2 ** 64 - 1
    # what the raw rollout attach refuses, the coded one refuses with the same message
    for args in ((None, 0, 0, 4096, 64, M64), (None, 0, 16385, 4096, 64, M64), (None, 0, 21, 4096, 4050, M64),
                 (None, 0, 21, 1 << 31, 64, M64), (None, 0, 21, 4096, -1, M64)):
        assert lib.b2rl_dedup_attach_rollouts(*args) == -1, args
        raw = lib.b2rl_last_error()
        assert lib.b2rl_dedup_attach_rollouts_coded(*args, 7072 * 5000) == -1, args
        assert lib.b2rl_last_error() == raw, (args, raw, lib.b2rl_last_error())
    bad = [((None, 0, 21, 4096, 64, M64, 0), b"pool_bytes must be positive"),
           ((None, 0, 21, 4096, 64, M64, 7072 * 200 + 8), b"multiple of 16"),
           ((None, 0, 21, 4096, 64, M64, 7072 * 149), b"window + 2 + frames_per_record"),
           ((None, 0, 21, 4096, 64, M64, 7072 * 150), b"null handle")]
    for args, msg in bad:
        assert lib.b2rl_dedup_attach_rollouts_coded(*args) == -1, args
        assert msg in lib.b2rl_last_error(), (args, lib.b2rl_last_error())
    A = 0x1000
    assert lib.b2rl_dedup_stage_rollouts(None, A, 32, A, A, None) == -1
    assert b"null handle" in lib.b2rl_last_error()
    assert lib.b2rl_launch_count() == launches


def test_store_signature_and_frame_source_refusals():
    import inspect
    from distributed_rl_b200 import replay as R
    sig = inspect.signature(R.RolloutDedupReplay.__init__).parameters
    assert sig["pool_bytes"].default is None and issubclass(R.RolloutDedupReplay, R.StripDedupReplay)
    coded, raw = types.SimpleNamespace(coded=True), types.SimpleNamespace(coded=False)
    with pytest.raises(ValueError, match="encoded"):
        R.RolloutDedupReplay.frame_source(coded, "state")
    with pytest.raises(KeyError, match="next_state"):
        R.RolloutDedupReplay.frame_source(coded, "next_state")
    with pytest.raises(ValueError, match="coded frame pool"):
        R.RolloutDedupReplay.stage_frames(raw, None, {})
