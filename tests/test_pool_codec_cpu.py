"""CPU tests of the compressed R2D2 frame pool (R2D2Config.POOL_CODEC, DESIGN.md §4.21): the numpy restatement of the
codec (tests/pool_codec_model.py) on random, constant, synthetic Atari-like and hand-built frames with pinned bytes;
the synthetic frame source; the unit-ring model of the store against the frame-only model; the configuration keys
and their refusals; and the new entry points' refusals before any CUDA work."""
import ctypes
import importlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pool_codec_model as M                                   # noqa: E402
from strip_dedup_model import StripDedupModel, max_batch      # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _roundtrip(f):
    e = M.encode(f)
    assert e.dtype == np.uint8 and len(e) % 16 == 0 and 16 <= len(e) <= M.RAW_BYTES
    assert int(e[1]) | int(e[2]) << 8 == len(e) // 16
    np.testing.assert_array_equal(M.decode(e), f)
    np.testing.assert_array_equal(M.encode(f.copy()), e)           # deterministic
    return e


def test_random_frames_are_stored_raw():
    rng = np.random.default_rng(1)
    for _ in range(8):
        f = rng.integers(0, 256, (84, 84), dtype=np.uint8)
        e = _roundtrip(f)
        assert len(e) == 7072 and e[0] == M.RAW
        np.testing.assert_array_equal(e[16:], f.ravel())
        assert not e[3:16].any()


def test_constant_frames_take_the_minimum():
    for v in (0, 1, 142, 255):
        f = np.full((84, 84), v, np.uint8)
        e = _roundtrip(f)
        # header + one coded row's mask + one literal = 28 bytes: two units
        assert len(e) == 32 and e[0] == M.ROWRUN
        assert e[16:27].tolist() == [1] + [0] * 10 and e[27] == v and not e[28:].any()


@pytest.mark.parametrize("r,x", [(0, 0), (0, 83), (83, 0), (83, 83), (41, 0), (41, 83), (0, 41), (83, 41)])
def test_a_single_changed_pixel(r, x):
    f = np.full((84, 84), 7, np.uint8)
    f[r, x] = 200
    e = _roundtrip(f)
    assert e[0] == M.ROWRUN
    coded = 1 + (r > 0) + (r < 83)            # row 0, the changed row, and the row after it
    assert 84 - int(np.unpackbits(e[3:14], bitorder="little").sum()) == coded
    assert len(e) == 16 * -(-(16 + 11 * coded + _literals(f)) // 16)


def _literals(f):
    rep = np.zeros(84, bool)
    rep[1:] = (f[1:] == f[:-1]).all(1)
    ch = np.ones((84, 84), bool)
    ch[:, 1:] = f[:, 1:] != f[:, :-1]
    return int(ch[~rep].sum())


def test_long_chains_of_repeated_rows_and_alternating_pixels():
    f = np.zeros((84, 84), np.uint8)
    f[:, ::2] = 255
    e = _roundtrip(f)                          # every row repeats row 0: one coded row of 84 literals
    assert e[0] == M.ROWRUN and len(e) == 16 * -(-(16 + 11 + 84) // 16)
    g = np.zeros((84, 84), np.uint8)
    g[::2, ::2] = g[1::2, 1::2] = 255          # a checkerboard: no row repeats, 84 literals a row
    e = _roundtrip(g)
    assert e[0] == M.RAW and len(e) == 7072     # 16 + 84 (11 + 84) bytes is more than raw
    h = np.repeat(np.arange(84, dtype=np.uint8)[:, None] // 21, 84, axis=1)   # four bands of 21 equal rows
    e = _roundtrip(h)
    assert e[0] == M.ROWRUN and len(e) == 16 * -(-(16 + 4 * 12) // 16)


def test_pinned_bytes_of_hand_built_frames():
    f = np.zeros((84, 84), np.uint8)
    f[0, 0] = 9
    f[1:, 80:] = 3
    e = M.encode(f)
    # rows: 0 coded (pixels 9 at x=0, then 0 from x=1), 1 coded (0, then 3 from x=80), 2..83 repeat row 1
    expect = [1, 3, 0] + [0b11111100, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0x0F] + [0, 0]
    expect += [0x03] + [0] * 10                      # row 0's change mask: x = 0, 1
    expect += [0x01] + [0] * 9 + [0x01]              # row 1's: x = 0, 80
    expect += [9, 0, 0, 3]                           # literals
    expect += [0] * (48 - len(expect))              # 42 bytes: three units
    assert e.tolist() == expect
    g = np.arange(84 * 84, dtype=np.int64).reshape(84, 84).astype(np.uint8)
    e = M.encode(g)
    assert e[:16].tolist() == [0, 0xBA, 0x01] + [0] * 13 and e[16:].tolist() == g.ravel().tolist()


def test_synthetic_frames_round_trip_and_compress():
    sizes = []
    for ep in range(3):
        for k in (0, 1, 2, 50, 199):
            f = M.atari_frame(k, ep)
            np.testing.assert_array_equal(f, M.atari_frame(k, ep))       # deterministic
            e = _roundtrip(f)
            sizes.append(len(e))
    assert max(sizes) < 2000, sizes          # synthetic frames: well under the raw 7 072 bytes
    assert not np.array_equal(M.atari_frame(3, 0), M.atari_frame(4, 0))   # it moves every step


def test_synthetic_sequences_follow_the_actor_structure():
    T = 16
    strips, a, r, h0, h1, nd, kind = M.atari_sequences(24, T=T, actors=2, episode=(30, 60), seed=3, hidden=8)
    assert strips.shape == (24, T + 3, 84, 84) and strips.dtype == np.uint8
    again = M.atari_sequences(24, T=T, actors=2, episode=(30, 60), seed=3, hidden=8)[0]
    np.testing.assert_array_equal(strips, again)
    assert kind[0] == "first" and "mid" in kind
    for i, k in enumerate(kind):                     # a first strip opens with o_0 four times
        if k == "first":
            for j in range(1, 4):
                np.testing.assert_array_equal(strips[i, j], strips[i, 0])
    assert all(x == (0.0 if k == "done" else x) for k, x in zip(kind, nd.tolist()))
    assert all(x == 1.0 for k, x in zip(kind, nd.tolist()) if k == "mid")


def _stream(n, T, seed):
    return M.atari_sequences(n, T=T, actors=3, episode=(30, 70), seed=seed, hidden=8)


def test_unit_ring_model_equals_the_frame_model_with_a_large_pool():
    T, cap, F, W = 12, 24, 400, 48
    P = (F + 1) * M.RAW_UNITS
    strips, *_ = _stream(90, T, 5)
    prio = np.linspace(0.1, 2.0, 90).astype(np.float32)
    a, b = StripDedupModel(cap, F, W, T), M.CodedStripDedupModel(cap, F, W, T, P)
    assert M.coded_max_batch(cap, F, W, T + 3, P) == max_batch(cap, F, W, T + 3)
    for i in range(0, 90, 7):
        a.push(strips[i:i + 7], prio[i:i + 7])
        b.push(strips[i:i + 7], prio[i:i + 7])
        np.testing.assert_array_equal(a.planes, b.planes)
        np.testing.assert_array_equal(a.prio, b.prio)
        np.testing.assert_array_equal(a.live_slots(), b.live_slots())
        assert a.head == b.head
    assert b.head > F and 0 < b.units < b.P            # the frame ring wrapped; the unit ring, sized raw, never binds
    np.testing.assert_array_equal(b.strips(b.live_slots()), a.strips(a.live_slots()))


def test_unit_ring_model_when_the_byte_rule_binds():
    T, cap, F, W = 12, 200, 4000, 32
    strips, *_ = _stream(160, T, 7)
    mean_units = np.mean([M.units(f) for f in strips[:20].reshape(-1, 84, 84)])
    P = int((W + 2 + 2 * (T + 3)) * M.RAW_UNITS)      # room for the window and 2 sequences of raw frames
    prio = np.ones(160, np.float32)
    m, plain = M.CodedStripDedupModel(cap, F, W, T, P), StripDedupModel(cap, F, W, T)
    assert M.coded_max_batch(cap, F, W, T + 3, P) == 2
    wrapped = False
    for i in range(0, 160, 2):
        m.push(strips[i:i + 2], prio[i:i + 2])
        plain.push(strips[i:i + 2], prio[i:i + 2])
        np.testing.assert_array_equal(m.planes, plain.planes)       # the ids are the frame rule's
        wrapped |= m.units > P
        live = m.live_slots()
        assert len(live) <= len(plain.live_slots())
        # every live slot's strips decode to the pushed sequences
        first = (i + 2) - len(live)
        np.testing.assert_array_equal(m.strips(live), strips[first:i + 2])
        assert (m.units - m.uins[live] < P - (W + 1) * M.RAW_UNITS).all()
        assert (m.prio[np.setdiff1d(np.arange(cap), live)] == 0).all()
    assert wrapped and mean_units < M.RAW_UNITS / 3
    assert len(m.live_slots()) < len(plain.live_slots())            # the byte rule bound


def test_unit_ring_model_never_straddles_and_stays_within_the_units():
    T, cap, F, W = 8, 40, 900, 16
    strips, *_ = _stream(120, T, 11)
    rng = np.random.default_rng(0)
    strips[::9, 5] = rng.integers(0, 256, (len(strips[::9]), 84, 84), dtype=np.uint8)   # some raw frames
    P = (W + 2 + 2 * (T + 3)) * M.RAW_UNITS + 37     # not a multiple of any frame's length
    m = M.CodedStripDedupModel(cap, F, W, T, P)
    for i in range(0, 120, 2):
        m.push(strips[i:i + 2], np.ones(2, np.float32))
        live = m.live_slots()
        ent = np.unique(m.planes[live])
        assert ((m.foff[ent] % P) + m.flen[ent] <= P).all()
        np.testing.assert_array_equal(m.strips(live), strips[i + 2 - len(live):i + 2])
    assert m.units > P


# ---- configuration and entry points ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from distributed_rl_b200 import build, _lib
    build.build()
    return _lib.load()


def _configuration(tmp_path, monkeypatch, **extra):
    from distributed_rl_b200 import r2d2
    cfg = {"ALG": "R2D2", "FIXED_TRAJECTORY": 80, "MEM": 20, "USE_RESCALING": True, "ALPHA": 0.9, "BETA": 0.4,
           "TARGET_FREQUENCY": 2500, "N": 32, "GAMMA": 0.997, "BATCHSIZE": 32, "ACTION_SIZE": 6, "UNROLL_STEP": 5,
           "REPLAY_MEMORY_LEN": 1000, "REDIS_SERVER": "localhost", "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0",
           "BUFFER_SIZE": 100, "optim": {"name": "adam", "lr": 1e-4, "eps": 0.001}, "model": {}, **extra}
    path = tmp_path / "r2d2.json"
    path.write_text(json.dumps(cfg))
    monkeypatch.setenv("B2RL_CFG", str(path))
    monkeypatch.chdir(tmp_path)
    monkeypatch.syspath_prepend(os.path.join(REPO, "dropin"))
    sys.modules.pop("configuration", None)
    try:
        importlib.import_module("configuration")
        return r2d2.R2D2Config.from_configuration()
    finally:
        sys.modules.pop("configuration", None)


def test_pool_codec_keys_defaults_and_refusals(tmp_path, monkeypatch):
    from distributed_rl_b200 import r2d2, apex, impala
    assert r2d2.R2D2Config.POOL_CODEC is False and r2d2.R2D2Config.POOL_BYTES_PER_SEQUENCE is None
    c = r2d2.R2D2Config(FRAME_DEDUP=True, POOL_CODEC=True, REPLAY_MEMORY_LEN=10_000)
    F, W = r2d2.dedup_geometry(c)
    assert (F, W) == (480_000, 16_384) and r2d2.pool_bytes(c) == (F + 1) * 7072
    assert r2d2.pool_bytes(r2d2.R2D2Config(FRAME_DEDUP=True)) is None
    c2 = r2d2.R2D2Config(FRAME_DEDUP=True, POOL_CODEC=True, REPLAY_MEMORY_LEN=10_000, POOL_BYTES_PER_SEQUENCE=70_001.5)
    assert r2d2.pool_bytes(c2) == (700_015_000 // 16) * 16
    with pytest.raises(ValueError, match="POOL_CODEC"):
        r2d2.R2D2Config(POOL_CODEC=True)
    with pytest.raises(ValueError, match="POOL_CODEC"):
        r2d2.R2D2Config(FRAME_DEDUP=True, POOL_CODEC=True, HOST_POOL=True)
    with pytest.raises(ValueError, match="POOL_BYTES_PER_SEQUENCE"):
        r2d2.R2D2Config(FRAME_DEDUP=True, POOL_BYTES_PER_SEQUENCE=1000.0)
    with pytest.raises(ValueError, match="POOL_BYTES_PER_SEQUENCE"):
        r2d2.R2D2Config(FRAME_DEDUP=True, POOL_CODEC=True, POOL_BYTES_PER_SEQUENCE=0)
    for cls in (apex.ApexConfig, impala.ImpalaConfig):           # their captured steps read the pool in place
        assert "POOL_CODEC" not in cls.__dataclass_fields__
    got = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True, POOL_CODEC=True, POOL_BYTES_PER_SEQUENCE=60000)
    assert got.FRAME_DEDUP and got.POOL_CODEC and got.POOL_BYTES_PER_SEQUENCE == 60000
    plain = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True)
    assert not plain.POOL_CODEC and plain.POOL_BYTES_PER_SEQUENCE is None
    with pytest.raises(ValueError, match="POOL_CODEC"):
        _configuration(tmp_path, monkeypatch, POOL_CODEC=True)


def test_entry_points_refuse_bad_arguments_before_any_cuda_work(lib):
    from distributed_rl_b200 import _lib
    for s in ("b2rl_dedup_attach_strips_coded", "b2rl_dedup_codec_stats", "b2rl_frame_encode", "b2rl_frame_decode"):
        assert s in _lib.SIGNATURES
    mask = (1 << 63) - 1
    launches = lib.b2rl_launch_count()
    big = 7072 * (512 + 2 + 83)
    cases = (
        ((None, 0, 83, 4096, 512, mask, big), b"null handle"),
        ((None, 0, 83, 4096, 512, mask, 0), b"pool_bytes must be positive"),
        ((None, 0, 83, 4096, 512, mask, -16), b"pool_bytes must be positive"),
        ((None, 0, 83, 4096, 512, mask, big + 8), b"multiple of 16"),
        ((None, 0, 83, 4096, 512, mask, big - 16), b"one record beyond the window"),
        ((None, 0, 2, 4096, 512, mask, big), b"frames_per_record must"),
        ((None, 0, 83, 595, 512, mask, big), b"pool_frames - window"),
    )
    for args, msg in cases:
        assert lib.b2rl_dedup_attach_strips_coded(*args) == -1, args    # B2RL_ERR_INVALID
        assert msg in lib.b2rl_last_error(), (args, lib.b2rl_last_error())
    u = ctypes.c_int64(-1)
    assert lib.b2rl_dedup_codec_stats(None, ctypes.byref(u), None, None) == -1 and u.value == -1
    assert lib.b2rl_frame_encode(None, -1, None, None, None) == -1
    assert lib.b2rl_frame_encode(None, 1, None, None, None) == -1 and b"null" in lib.b2rl_last_error()
    assert lib.b2rl_frame_decode(None, 1, None, None) == -1 and b"null" in lib.b2rl_last_error()
    assert lib.b2rl_frame_encode(None, 0, None, None, None) == 0 and lib.b2rl_frame_decode(None, 0, None, None) == 0
    assert lib.b2rl_launch_count() == launches


def test_strip_store_signature_and_frame_source_refusal():
    import inspect
    import torch
    from distributed_rl_b200 import replay as R
    assert inspect.signature(R.StripDedupReplay.__init__).parameters["pool_bytes"].default is None
    assert "pool_bytes" not in inspect.signature(R.DedupReplay.__init__).parameters
    pool = torch.zeros(4096, dtype=torch.uint8)          # a coded pool is a flat byte ring, not (F, 84, 84) frames
    with pytest.raises(ValueError, match="encoded"):
        R._frame_source(R.PlaneFrames(pool, torch.zeros(32, dtype=torch.int32), 0, 1))


def test_codec_helpers_refuse_anything_but_device_uint8_rows():
    import torch
    from distributed_rl_b200 import replay as R
    cases = ((R.encode_frames, torch.zeros(2, 84, 84, dtype=torch.uint8)),              # host memory
             (R.encode_frames, torch.zeros(2, 84, 84, dtype=torch.int32)),
             (R.decode_frames, torch.zeros(2, 7072, dtype=torch.uint8)),
             (R.decode_frames, [0] * 7072))
    for fn, x in cases:
        with pytest.raises(ValueError, match="CUDA uint8"):
            fn(x)
