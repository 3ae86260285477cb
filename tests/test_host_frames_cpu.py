"""CPU checks of R2D2 host frames (R2D2Config.HOST_FRAMES): the config key and its drop-in `configuration` key, the
refusal of PAYLOAD_POOL beside it, the bytes each sequence keeps on the host and on the device, and the C ABI's refusal
of a host field whose rows are not whole 16-byte units, made before any CUDA call."""
import ctypes
import os
import subprocess
import sys
import textwrap

import pytest

from test_frame_strips_cpu import REPO, _r2d2_cfg_json


def test_the_config_key_defaults_to_hbm():
    from distributed_rl_b200.r2d2 import R2D2Config
    assert R2D2Config().HOST_FRAMES is False
    assert R2D2Config(HOST_FRAMES=True, FRAME_STRIP=True).HOST_FRAMES is True


def test_payload_pool_is_refused_with_host_frames():
    from distributed_rl_b200.r2d2 import R2D2Config
    with pytest.raises(ValueError, match="HOST_FRAMES.*PAYLOAD_POOL"):
        R2D2Config(HOST_FRAMES=True, PAYLOAD_POOL=16)
    R2D2Config(PAYLOAD_POOL=16)                                 # the benchmark stand-in alone is unchanged


@pytest.mark.parametrize("value", [None, False, True])
def test_the_dropin_configuration_key(tmp_path, value):
    _r2d2_cfg_json(tmp_path, **({} if value is None else {"HOST_FRAMES": value, "FRAME_STRIP": True}))
    code = """
        import configuration as C
        from distributed_rl_b200.r2d2 import R2D2Config
        print("HOST", C.HOST_FRAMES, R2D2Config.from_configuration().HOST_FRAMES)
    """
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(REPO, "dropin"), REPO]))
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=tmp_path, env=env, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    want = bool(value)
    assert f"HOST {want} {want}" in r.stdout


@pytest.mark.parametrize("strip, host_bytes", [(True, 585_648), (False, 2_257_920)])
def test_bytes_per_sequence_on_the_host_and_on_the_device(strip, host_bytes):
    """The frames go to the host, the five small fields (action, reward, h0, h1, notdone) stay in HBM; the host rows
    are whole 16-byte units, as the host-row gather needs."""
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.r2d2 import R2D2Config
    fields = R.r2d2_config_fields(R2D2Config(FRAME_STRIP=strip, HOST_FRAMES=True))
    on_host = [f for f in fields if f.name == "state"]
    on_device = [f for f in fields if f.name != "state"]
    assert sum(f.nbytes for f in on_host) == host_bytes and host_bytes % 16 == 0
    assert sum(f.nbytes for f in on_device) == 4_740
    if strip:   # 2^20 sequences: about 5 GB of small fields on the card, 614 GB of strips pinned on the host
        assert round((1 << 20) * 4_740 / 1e9, 1) == 5.0 and round((1 << 20) * host_bytes / 1e9) == 614


@pytest.fixture(scope="module")
def lib():
    from distributed_rl_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.mark.parametrize("row_bytes", [1, 8, 4740, 585_648 + 8])
def test_a_host_field_of_partial_16_byte_units_is_refused(lib, row_bytes):
    from distributed_rl_b200._lib import MAX_FIELDS, ReplayDesc
    d = ReplayDesc()
    d.capacity, d.n_fields, d.device = 4, 2, 0
    d.field_bytes[0], d.field_bytes[1] = 16, row_bytes
    on_host = (ctypes.c_int32 * MAX_FIELDS)(0, 1)
    h = ctypes.c_void_p()
    assert lib.b2rl_replay_create_placed(ctypes.byref(d), on_host, ctypes.byref(h)) == -1   # B2RL_ERR_INVALID
    assert b"16-byte" in lib.b2rl_last_error() and not h.value


def test_the_placement_entry_points_refuse_null_arguments(lib):
    assert lib.b2rl_replay_create_placed(None, None, None) < 0
    assert b"null" in lib.b2rl_last_error()
    assert lib.b2rl_replay_field_placement(None, 0, None) < 0
    assert b"null" in lib.b2rl_last_error()


def test_device_replay_refuses_unknown_host_fields(lib):
    import torch
    from distributed_rl_b200 import replay as R
    if torch.cuda.is_available():
        pytest.skip("GPU present; covered by the gpu tests")
    with pytest.raises((ValueError, RuntimeError, AssertionError)):
        R.DeviceReplay(4, R.r2d2_fields(8, strip=True), "cuda:0", host_fields=("frames",))
