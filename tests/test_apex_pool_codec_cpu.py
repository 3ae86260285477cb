"""CPU tests of the coded Ape-X frame pool (ApexConfig.FRAME_CODEC, R.CodedDedupReplay, DESIGN.md §4.22): the store's
model is the unit-ring strip model with T = 5, fed s and s' side by side (R = 8), checked against the frame-only
Ape-X model and with the byte rule binding past several wraps; the synthetic Player-like records; the configuration
keys, defaults and refusals; and the refusals of the new entry point and of conv_1's coded frame source before any
CUDA work."""
import ctypes
import importlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pool_codec_model as M                                   # noqa: E402
from apex_atari_records import atari_records                  # noqa: E402
from dedup_model import DedupModel                            # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from distributed_rl_b200 import build, _lib
    build.build()
    return _lib.load()


def _pairs(s, ns):
    return np.concatenate([s, ns], axis=1)                     # (n, 8, 84, 84): planes 0-3 of s, 4-7 of s'


def test_records_are_player_like():
    s, ns, a, r, d = atari_records(200, actors=4, unroll=3, seed=1)
    assert s.shape == ns.shape == (200, 4, 84, 84) and s.dtype == np.uint8
    assert np.array_equal(s[0, 0], s[0, 3])                    # an episode starts with its first frame four times
    # s' of a record is the stack UNROLL_STEP steps later of the same actor: with chunk 5 and 4 actors, record t of
    # an actor's first chunk pairs with record t + 3 of that chunk
    assert np.array_equal(ns[0], s[3]) and np.array_equal(ns[1], s[4])
    new = [len({f.tobytes() for f in _pairs(s[:k], ns[:k]).reshape(-1, 84 * 84)}) for k in (100, 200)]
    assert new[1] - new[0] < 2 * 100                           # about one new frame per record


def test_model_with_a_large_ring_gives_the_frame_models_ids():
    cap, F, W = 64, 400, 48
    P = (F + 1) * M.RAW_UNITS
    s, ns, *_ = atari_records(300, seed=2)
    prio = np.linspace(0.1, 2.0, 300).astype(np.float32)
    a, b = DedupModel(cap, F, W), M.CodedStripDedupModel(cap, F, W, 5, P)
    assert b.R == 8
    for i in range(0, 300, 9):
        a.push(s[i:i + 9], ns[i:i + 9], prio[i:i + 9])
        b.push(_pairs(s[i:i + 9], ns[i:i + 9]), prio[i:i + 9])
        np.testing.assert_array_equal(a.planes.reshape(cap, 8), b.planes)
        np.testing.assert_array_equal(a.prio, b.prio)
        np.testing.assert_array_equal(a.live_slots(), b.live_slots())
        assert a.head == b.head
    assert b.head > F and 0 < b.units < b.P
    live = b.live_slots()
    ss, nn = a.stacks(live)
    np.testing.assert_array_equal(b.strips(live), _pairs(ss, nn))


def test_model_with_the_byte_rule_binding_past_several_wraps():
    cap, F, W = 256, 4000, 16
    s, ns, *_ = atari_records(1200, seed=3)
    P = (W + 2 + 8 * 2) * M.RAW_UNITS                          # the window and two records of raw frames
    m, plain = M.CodedStripDedupModel(cap, F, W, 5, P), DedupModel(cap, F, W)
    assert M.coded_max_batch(cap, F, W, 8, P) == 2
    prio = np.ones(1200, np.float32)
    for i in range(0, 1200, 2):
        m.push(_pairs(s[i:i + 2], ns[i:i + 2]), prio[i:i + 2])
        plain.push(s[i:i + 2], ns[i:i + 2], prio[i:i + 2])
        np.testing.assert_array_equal(m.planes, plain.planes.reshape(cap, 8))   # ids are the frame rule's
        live = m.live_slots()
        first = i + 2 - len(live)
        if i % 20 == 0 or i == 1198:                                                # nothing overwritten
            np.testing.assert_array_equal(m.strips(live), _pairs(s[first:i + 2], ns[first:i + 2]))
        ent = np.unique(m.planes[live])
        assert ((m.foff[ent] % P) + m.flen[ent] <= P).all()                       # nothing straddles
        assert (m.units - m.uins[live] < P - (W + 1) * M.RAW_UNITS).all()
    assert m.units > 3 * P
    assert len(m.live_slots()) < len(plain.live_slots())


def _configuration(tmp_path, monkeypatch, **extra):
    from distributed_rl_b200 import apex
    cfg = {"ALG": "APE_X", "ALPHA": 0.6, "BETA": 0.4, "TARGET_FREQUENCY": 2500, "N": 32, "GAMMA": 0.99, "BATCHSIZE": 32,
           "ACTION_SIZE": 6, "UNROLL_STEP": 3, "REPLAY_MEMORY_LEN": 1000, "REDIS_SERVER": "localhost",
           "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0", "BUFFER_SIZE": 100,
           "optim": {"name": "rmsprop", "lr": 1e-4, "eps": 0.001}, "model": {}, **extra}
    path = tmp_path / "cfg.json"
    path.write_text(json.dumps(cfg))
    monkeypatch.setenv("B2RL_CFG", str(path))
    monkeypatch.chdir(tmp_path)
    monkeypatch.syspath_prepend(os.path.join(REPO, "dropin"))
    sys.modules.pop("configuration", None)
    try:
        importlib.import_module("configuration")
        return apex.ApexConfig.from_configuration()
    finally:
        sys.modules.pop("configuration", None)


def test_frame_codec_keys_defaults_and_refusals(tmp_path, monkeypatch):
    from distributed_rl_b200 import apex
    assert apex.ApexConfig.FRAME_CODEC is False and apex.ApexConfig.POOL_BYTES_PER_TRANSITION is None
    assert "POOL_CODEC" not in apex.ApexConfig.__dataclass_fields__     # R2D2's staged form stays R2D2's
    a = apex.ApexConfig(FRAME_DEDUP=True, FRAME_CODEC=True, REPLAY_MEMORY_LEN=1 << 21)
    F, W = apex.dedup_geometry(a)
    assert (F, W) == (1 << 23, 1 << 20) and apex.pool_bytes(a) == (F + 1) * 7072
    assert apex.pool_bytes(apex.ApexConfig(FRAME_DEDUP=True)) is None
    a2 = apex.ApexConfig(FRAME_DEDUP=True, FRAME_CODEC=True, REPLAY_MEMORY_LEN=1000, POOL_BYTES_PER_TRANSITION=700.7)
    assert apex.pool_bytes(a2) == 700_700 // 16 * 16
    with pytest.raises(ValueError, match="FRAME_CODEC.*FRAME_DEDUP"):
        apex.ApexConfig(FRAME_CODEC=True)
    with pytest.raises(ValueError, match="POOL_BYTES_PER_TRANSITION"):
        apex.ApexConfig(FRAME_DEDUP=True, POOL_BYTES_PER_TRANSITION=1000.0)
    with pytest.raises(ValueError, match="POOL_BYTES_PER_TRANSITION"):
        apex.ApexConfig(FRAME_DEDUP=True, FRAME_CODEC=True, POOL_BYTES_PER_TRANSITION=0)
    got = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True, FRAME_CODEC=True,
                         POOL_BYTES_PER_TRANSITION=2000)
    assert got.FRAME_DEDUP and got.FRAME_CODEC and got.POOL_BYTES_PER_TRANSITION == 2000
    plain = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True)
    assert not plain.FRAME_CODEC and plain.POOL_BYTES_PER_TRANSITION is None
    with pytest.raises(ValueError, match="FRAME_CODEC"):
        _configuration(tmp_path, monkeypatch, FRAME_CODEC=True)


def test_entry_points_refuse_bad_arguments_before_any_cuda_work(lib):
    from distributed_rl_b200 import _lib
    assert "b2rl_dedup_attach_coded" in _lib.SIGNATURES and "b2rl_dedup_coded_offsets" in _lib.SIGNATURES
    launches = lib.b2rl_launch_count()
    bad = [((None, 0, 1024, 64, ~0 & (2 ** 64 - 1), 0), b"pool_bytes must be positive"),
           ((None, 0, 1024, 64, 0, 7072 * 80 + 8), b"multiple of 16"),
           ((None, 0, 1024, 64, 0, 7072 * 73), b"window + 10"),
           ((None, 0, 1024, 1020, 0, 7072 * 2000), b"pool_frames - window > 8"),
           ((None, 0, 1 << 31, 64, 0, 7072 * 2000), b"below 2^31"),
           ((None, 0, 1024, 64, 0, 7072 * 74), b"null handle")]
    for args, msg in bad:
        assert lib.b2rl_dedup_attach_coded(*args) == -1, args
        assert msg in lib.b2rl_last_error(), (args, lib.b2rl_last_error())
    p = ctypes.c_void_p(1)
    assert lib.b2rl_dedup_coded_offsets(None, ctypes.byref(p)) == -1 and p.value == 1
    assert lib.b2rl_launch_count() == launches


def test_conv1_refuses_a_malformed_coded_source(lib):
    from distributed_rl_b200 import _lib
    A = 0x1000
    good = dict(pool=A, planes=A, offsets=A, rows=8, pool_units=442, pool_frames=64)
    fwd = lambda **kw: lib.b2rl_conv1_fused(ctypes.byref(_lib.Frames(**(good | kw))), None, 8, A, A, 1, 32, A, 0, None)
    wgrad = lambda **kw: lib.b2rl_conv1_wgrad(ctypes.byref(_lib.Frames(**(good | kw))), None, 8, A, None, 32, A, A, 0,
                                              None)
    launches = lib.b2rl_launch_count()
    for kw, msg in (({"plane_stride": 1}, b"plane_stride 0 or 8"), ({"plane_stride": 4}, b"plane_stride 0 or 8"),
                    ({"pool_units": 0}, b"positive pool_units"), ({"pool_frames": -1}, b"positive pool_units"),
                    ({"pool_frames": 1 << 31}, b"below 2^31"), ({"plane_base": 2}, b"plane_base"),
                    ({"offsets": A + 4}, b"8-byte aligned"), ({"pool": A + 8}, b"16-byte aligned"),
                    ({"pool": None}, b"null frame pool"), ({"base": A}, b"exactly one")):
        for fn in (fwd, wgrad):
            assert fn(**kw) == -1, kw
            assert msg in lib.b2rl_last_error(), (kw, lib.b2rl_last_error())
    assert lib.b2rl_launch_count() == launches


def test_coded_store_signature_and_frame_source_refusals():
    import inspect
    import torch
    from distributed_rl_b200 import replay as R
    sig = inspect.signature(R.CodedDedupReplay.__init__).parameters
    assert list(sig)[:5] == ["self", "capacity", "pool_frames", "window", "pool_bytes"]
    assert sig["hash_mask"].default == R.DEDUP_HASH_MASK and issubclass(R.CodedDedupReplay, R.DedupReplay)
    assert "pool_bytes" not in inspect.signature(R.DedupReplay.__init__).parameters
    pool, planes = torch.zeros(4096, dtype=torch.uint8), torch.zeros(64, dtype=torch.int32)
    offsets = torch.zeros(16, dtype=torch.int64)
    with pytest.raises(ValueError, match="encoded"):                       # a plain PlaneFrames over a flat ring
        R._frame_source(R.PlaneFrames(pool, planes, 0))
    with pytest.raises(ValueError, match="on the GPU"):                     # host tensors
        R._frame_source(R.CodedPlaneFrames(pool, planes, offsets, 16, 0))
    with pytest.raises(ValueError, match="flat uint8 ring"):
        R._frame_source(R.CodedPlaneFrames(torch.zeros(64, 64, dtype=torch.uint8), planes, offsets, 16, 0))
    assert R.CodedPlaneFrames(pool, planes, offsets, 16, 4).rows == 8
