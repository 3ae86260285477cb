"""CPU tests of the host-placed frame pool of the deduplicated R2D2 store (R2D2Config.HOST_POOL, DESIGN.md §4.19): the
configuration key and its refusals, the new entry points' refusals before any CUDA work, and conv_1's refusal of a
plane table over a pool in host memory."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def test_host_pool_key_default_and_refusals(tmp_path, monkeypatch):
    from distributed_rl_b200 import r2d2
    assert r2d2.R2D2Config.HOST_POOL is False and not r2d2.R2D2Config().HOST_POOL
    c = r2d2.R2D2Config(FRAME_DEDUP=True, HOST_POOL=True, REPLAY_MEMORY_LEN=10_000)
    assert c.FRAME_STRIP and r2d2.dedup_geometry(c) == (480_000, 16_384)     # the pool's geometry does not change
    with pytest.raises(ValueError, match="HOST_POOL"):
        r2d2.R2D2Config(HOST_POOL=True)
    with pytest.raises(ValueError, match="HOST_POOL"):
        r2d2.R2D2Config(HOST_POOL=True, HOST_FRAMES=True)
    for kw in (dict(HOST_FRAMES=True), dict(PAYLOAD_POOL=64), dict(HOST_POOL=True, HOST_FRAMES=True),
               dict(HOST_POOL=True, PAYLOAD_POOL=64)):
        with pytest.raises(ValueError, match="FRAME_DEDUP"):
            r2d2.R2D2Config(FRAME_DEDUP=True, **kw)
    got = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True, HOST_POOL=True)
    assert got.FRAME_DEDUP and got.HOST_POOL and got.FRAME_STRIP
    plain = _configuration(tmp_path, monkeypatch, FRAME_DEDUP=True)
    assert plain.FRAME_DEDUP and not plain.HOST_POOL
    with pytest.raises(ValueError, match="HOST_POOL"):
        _configuration(tmp_path, monkeypatch, HOST_POOL=True)


def test_entry_points_refuse_bad_arguments_before_any_cuda_work(lib):
    from distributed_rl_b200 import _lib
    assert "b2rl_dedup_attach_strips_placed" in _lib.SIGNATURES and "b2rl_dedup_pool_placement" in _lib.SIGNATURES
    mask = (1 << 63) - 1
    launches = lib.b2rl_launch_count()
    cases = (
        ((None, 0, 83, 4096, 512, mask, 1), b"null handle"),
        ((None, 0, 83, 4096, 512, mask, 2), b"pool_on_host must be 0 or 1"),
        ((None, 0, 83, 4096, 512, mask, -1), b"pool_on_host must be 0 or 1"),
        ((None, 0, 2, 4096, 512, mask, 1), b"frames_per_record must"),
        ((None, 0, 70000, 1 << 20, 512, mask, 1), b"frames_per_record must"),
        ((None, 0, 83, 595, 512, mask, 1), b"pool_frames - window"),
        ((None, 0, 83, 4096, -1, mask, 1), b"pool_frames - window"),
        ((None, 0, 83, 1 << 31, 512, mask, 1), b"2^31"),
    )
    for args, msg in cases:
        assert lib.b2rl_dedup_attach_strips_placed(*args) == -1, args    # B2RL_ERR_INVALID
        assert msg in lib.b2rl_last_error(), (args, lib.b2rl_last_error())
    flag, ptr = ctypes.c_int32(-1), ctypes.c_void_p()
    assert lib.b2rl_dedup_pool_placement(None, ctypes.byref(flag), ctypes.byref(ptr)) == -1    # B2RL_ERR_INVALID
    assert b"null" in lib.b2rl_last_error() and flag.value == -1
    assert lib.b2rl_launch_count() == launches


def test_pairs_layout_takes_no_host_pool():
    """Ape-X's store has no placed attach: its DedupReplay takes no host_pool; the strip store's defaults to HBM."""
    import inspect
    from distributed_rl_b200 import replay as R
    assert "host_pool" not in inspect.signature(R.DedupReplay.__init__).parameters
    assert inspect.signature(R.StripDedupReplay.__init__).parameters["host_pool"].default is False


def test_frame_source_refuses_a_plane_table_over_a_host_pool():
    from distributed_rl_b200 import replay as R
    pool = torch.zeros(16, 84, 84, dtype=torch.uint8)
    planes = torch.zeros(32, dtype=torch.int32)
    with pytest.raises(ValueError, match="host memory"):
        R._frame_source(R.PlaneFrames(pool, planes, 0, 1))
    with pytest.raises(ValueError, match="host memory"):
        R.conv1_fused(R.PlaneFrames(pool, planes, 0, 1), None, None)
