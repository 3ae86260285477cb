"""CPU checks of R2D2 frame strips (R2D2Config.FRAME_STRIP): a sequence of T observations stored as its T + 3 distinct
frames, stack t being frames t .. t + 3.  The encoding and its refusal of records that do not slide, the window and
stack views, the row arithmetic conv_1 and the served step rely on, the serve-ring layout of a strip record, the
drop-in configuration key, the refusals between strip and stack servers and learners, the reference-format `BATCH`
of the Redis-protocol server, and the sequences the unmodified reference actor sends (tests/golden/r2d2_actor.npz,
made by tests/golden/make_r2d2_actor_golden.py)."""
import dataclasses
import json
import os
import pickle
import subprocess
import sys
import textwrap
import threading
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from fake_redis import FakeRedis

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rs():
    from distributed_rl_b200 import build
    build.build()
    from distributed_rl_b200 import replay_server
    return replay_server


def _strips(n, T, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, T + 3, 84, 84), dtype=np.uint8)


def _stacks(strips):
    """The stacks of strips, built frame by frame: stack t of a sequence is its frames t .. t + 3."""
    n, T = strips.shape[0], strips.shape[1] - 3
    return np.stack([np.stack([strips[i, t:t + 4] for t in range(T)]) for i in range(n)])


def test_strip_encoding_round_trips_and_every_window_is_its_stack():
    from distributed_rl_b200 import replay as R
    n, T = 3, 12
    strips = _strips(n, T)
    stacks = _stacks(strips)
    np.testing.assert_array_equal(R.encode_strips(stacks), strips)
    np.testing.assert_array_equal(R.encode_strips(torch.from_numpy(stacks)), strips)
    st = torch.from_numpy(strips)
    win = R.strip_windows(st)
    assert win.shape == (n * (T + 3) - 3, 4, 84, 84) and win.stride() == (7056, 7056, 84, 1)
    assert win.data_ptr() == st.data_ptr()                          # zero-copy
    for s in range(n):
        for t in range(T):
            assert torch.equal(win[s * (T + 3) + t], torch.from_numpy(stacks[s, t]))
    view = R.strip_stacks(st)
    assert view.shape == (n, T, 4, 84, 84) and view.data_ptr() == st.data_ptr()
    assert torch.equal(view, torch.from_numpy(stacks))
    assert torch.equal(R.as_stacks(st), view) and R.as_stacks(view) is view
    back = R.stacks_strips(view)
    assert back.data_ptr() == st.data_ptr() and torch.equal(back, st)
    assert R.stacks_strips(torch.from_numpy(stacks)) is None        # materialised stacks are not a strip view
    sub = view[1:]                                                  # a slice of the view keeps its strips
    assert torch.equal(R.stacks_strips(sub), st[1:])


def _records(stacks, seed=0):
    """Reference-format R2D2 records (R2D2/Player.py:38-63,312-319): [(h0, h1), (s, a, r) x T, done, prio]."""
    rng = np.random.default_rng(seed)
    out = []
    for i, st in enumerate(stacks):
        h = (torch.from_numpy(rng.standard_normal((1, 1, 512)).astype(np.float32)),
             torch.from_numpy(rng.standard_normal((1, 1, 512)).astype(np.float32)))
        rec = [h]
        for t in range(st.shape[0]):
            rec += [st[t].copy(), int(rng.integers(0, 6)), float(rng.standard_normal())]
        rec += [bool(i % 2), float(rng.random())]
        arr = np.empty(len(rec), object)
        for j, v in enumerate(rec):
            arr[j] = v
        out.append(pickle.dumps(arr))
    return out


class _Store:
    def __init__(self):
        self.pushes = []

    def push(self, fields, p):
        self.pushes.append(([np.asarray(f).copy() for f in fields], np.asarray(p).copy()))


def _ingest(T, strip=True):
    """An r2d2.Replay reduced to its ingest: the store records what it is handed."""
    from distributed_rl_b200 import r2d2
    rp = object.__new__(r2d2.Replay)
    rp.cfg = r2d2.R2D2Config(FIXED_TRAJECTORY=T, FRAME_STRIP=strip, LEARNER_DEVICE="cpu")
    rp._lock, rp.store, rp.total_frame = threading.Lock(), _Store(), 0
    return rp


def test_records_are_pushed_as_strips():
    from distributed_rl_b200 import wire
    n, T = 4, 10
    strips = _strips(n, T, 1)
    stacks = _stacks(strips)
    blobs = _records(stacks)
    cols, p = wire.decode_r2d2([pickle.loads(b) for b in blobs], T, strip=True)
    np.testing.assert_array_equal(cols[0], strips)
    ref, pr = wire.decode_r2d2([pickle.loads(b) for b in blobs], T)
    np.testing.assert_array_equal(ref[0], stacks)
    for a, b in zip(cols[1:], ref[1:]):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(p, pr)
    rp = _ingest(T)
    rp.push_records(blobs)
    (fields, prio), = rp.store.pushes
    assert fields[0].shape == (n, T + 3, 84, 84)                    # the copy to the device carries the strips only
    np.testing.assert_array_equal(fields[0], strips)
    rp.push_arrays(stacks, *ref[1:], pr)                            # stacks are encoded
    rp.push_arrays(strips, *ref[1:], pr)                            # strips go as they are
    for fields, _ in rp.store.pushes[1:]:
        np.testing.assert_array_equal(fields[0], strips)
    assert rp.total_frame == 3 * n
    plain = _ingest(T, strip=False)
    plain.push_arrays(stacks, *ref[1:], pr)                         # without FRAME_STRIP nothing changes
    np.testing.assert_array_equal(plain.store.pushes[0][0][0], stacks)


@pytest.mark.parametrize("channel", [0, 1, 2])
def test_a_record_that_does_not_slide_is_refused_and_nothing_is_pushed(channel):
    from distributed_rl_b200 import wire
    n, T = 4, 10
    stacks = _stacks(_strips(n, T, 2))
    stacks[2, 5, channel] ^= 1                                      # one channel of one stack altered
    rp = _ingest(T)
    with pytest.raises(ValueError, match="record 2: stack [56] "):
        rp.push_arrays(stacks, np.zeros((n, T), np.int32), np.zeros((n, T), np.float32),
                       np.zeros((n, 512), np.float32), np.zeros((n, 512), np.float32), np.ones(n, np.float32),
                       np.ones(n, np.float32))
    with pytest.raises(ValueError, match="record 2: stack [56] "):
        rp.push_records(_records(stacks))
    with pytest.raises(ValueError, match="record 2"):
        wire.decode_r2d2([pickle.loads(b) for b in _records(stacks)], T, strip=True)
    assert rp.store.pushes == [] and rp.total_frame == 0
    stacks[2, 5, channel] ^= 1
    stacks[0, 0, 3] ^= 1            # the newest frame of a stack is free: it is stored, only the next stack must agree
    with pytest.raises(ValueError, match="record 0: stack 1 "):
        rp.push_records(_records(stacks))


def test_a_channel_change_in_the_newest_frame_is_stored():
    """Channel 3 of the last stack is seen by no later stack: any value slides."""
    from distributed_rl_b200 import replay as R
    T = 6
    strips = _strips(1, T, 3)
    stacks = _stacks(strips)
    stacks[0, T - 1, 3] = 7
    out = R.encode_strips(stacks)
    np.testing.assert_array_equal(out[0, T + 2], np.full((84, 84), 7, np.uint8))


def test_row_arithmetic_of_windows():
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.learner_common import time_major_rows
    T, B = 80, 5
    assert R.sequence_rows(B, T, False) == (T, B * T, 28224)
    assert R.sequence_rows(B, T, True) == (T + 3, B * (T + 3) - 3, 7056)
    seq = torch.tensor([7, 0, 3, 7, 2])                             # repeated slots are fine
    t_idx = torch.arange(T).view(T, 1)
    rows = time_major_rows(seq, t_idx, T + 3).view(T, B)
    for t in (0, 1, T - 1):
        assert rows[t].tolist() == [s * (T + 3) + t for s in seq.tolist()]
    assert torch.equal(time_major_rows(seq, t_idx), time_major_rows(seq, t_idx, T))
    for n in (1, 2, 9):                                             # the last window ends with the allocation
        _, rows_n, stride = R.sequence_rows(n, T, True)
        assert (rows_n - 1) * stride + 28224 == n * (T + 3) * 7056
        assert R.strip_windows(torch.zeros((n, T + 3, 84, 84), dtype=torch.uint8)).shape[0] == rows_n


@pytest.mark.parametrize("strip", [False, True])
def test_bind_covers_exactly_the_windows_of_the_slot(rs, strip):
    from distributed_rl_b200 import replay as R
    B, T = 4, 80
    fields = R.r2d2_fields(T, strip=strip)
    _, rows, stride = R.sequence_rows(B, T, strip)
    table = torch.zeros(2, dtype=torch.int64)
    _, to = rs.bind_targets(B, fields, {}, {"state": R.BoundFrames(table, 1, rows, stride)})
    assert to[0] == table.data_ptr() + 8
    for bad in (rows - 1, rows + 1):
        with pytest.raises(ValueError, match=f"{rows} frame rows {stride} bytes apart, not the {bad}"):
            rs.bind_targets(B, fields, {}, {"state": R.BoundFrames(table, 1, bad, stride)})
    other = 28224 if strip else 7056                                # the other layout's row stride
    with pytest.raises(ValueError, match="frame rows"):
        rs.bind_targets(B, fields, {}, {"state": R.BoundFrames(table, 1, rows, other)})


def test_ring_layout_of_a_strip_record(rs):
    from distributed_rl_b200 import replay as R
    fields = R.r2d2_fields(80, strip=True)
    fb = [f.nbytes for f in fields]
    assert fb == [83 * 7056, 320, 320, 2048, 2048, 4] and sum(fb) == 590_388
    assert sum(f.nbytes for f in R.r2d2_fields(80)) / sum(fb) > 3.83
    for batch in (1, 3, 32, 64):
        L = rs.serve_layout(batch, 4, fb)
        offs = [L.idx_off, L.w_off] + [L.field_off[i] for i in range(len(fb))]
        assert all(o % 16 == 0 for o in offs)
        for i in range(len(fb) - 1):                                # fields in record order, none overlapping
            assert L.field_off[i] + batch * fb[i] <= L.field_off[i + 1]
        assert L.field_off[len(fb) - 1] + 4 * batch <= L.slot_bytes and L.slot_bytes % 128 == 0
        if batch == 64:
            assert 37_700_000 < L.slot_bytes < 37_900_000           # 37.8 MB, against 144.8 MB for stacks


def _r2d2_cfg_json(tmp_path, **extra):
    from distributed_rl_b200.r2d2 import default_r2d2_model
    cfg = {"ALG": "R2D2", "REDIS_SERVER": "localhost", "ACTION_SIZE": 6, "ALPHA": 0.9, "BETA": 0.4, "GAMMA": 0.997,
           "TARGET_FREQUENCY": 2500, "N": 8, "BATCHSIZE": 32, "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0",
           "REPLAY_MEMORY_LEN": 10000, "BUFFER_SIZE": 1000, "UNROLL_STEP": 5, "FIXED_TRAJECTORY": 80, "MEM": 20,
           "USE_RESCALING": True, "optim": {"name": "adam", "lr": 1e-4, "eps": 0.001}, "model": default_r2d2_model(),
           **extra}
    (tmp_path / "cfg").mkdir(exist_ok=True)
    (tmp_path / "cfg" / "ape_x.json").write_text(json.dumps(cfg))


@pytest.mark.parametrize("value", [None, False, True])
def test_the_dropin_configuration_key(tmp_path, value):
    _r2d2_cfg_json(tmp_path, **({} if value is None else {"FRAME_STRIP": value}))
    code = """
        import configuration as C
        from distributed_rl_b200.r2d2 import R2D2Config
        print("STRIP", C.FRAME_STRIP, R2D2Config.from_configuration().FRAME_STRIP)
    """
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(REPO, "dropin"), REPO]))
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=tmp_path, env=env, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    want = bool(value)
    assert f"STRIP {want} {want}" in r.stdout


@pytest.mark.parametrize("learner_strip", [False, True])
def test_strip_and_stack_learners_and_servers_refuse_each_other(rs, monkeypatch, learner_strip):
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.learner_common import check_served_fused
    B = 8
    cfg = r2d2.R2D2Config(BATCHSIZE=B, SERVED_FUSED_STEP=True, FRAME_STRIP=learner_strip, LEARNER_DEVICE="cpu")
    server_fields = R.r2d2_fields(80, strip=not learner_strip)
    layout = rs.serve_layout(B, 2, [f.nbytes for f in server_fields])
    mem = SimpleNamespace(acquire=None, release=None, ring=SimpleNamespace(layout=layout))
    with pytest.raises(ValueError, match="record fields"):
        check_served_fused(cfg, mem, R.r2d2_config_fields(cfg))
    same = SimpleNamespace(acquire=None, release=None,
                           ring=SimpleNamespace(layout=rs.serve_layout(B, 2, [f.nbytes for f in R.r2d2_config_fields(cfg)])))
    check_served_fused(cfg, same, R.r2d2_config_fields(cfg))
    # the client compares the ring's field sizes with its config's before it maps any event
    conn = FakeRedis()
    conn.set(rs.RING_KEY, pickle.dumps({"handle": b"", "layout": bytes(layout), "device": 0}))
    monkeypatch.setattr(rs.ServeRing, "open", classmethod(lambda cls, h, lay, dev: SimpleNamespace(
        layout=type(layout).from_buffer_copy(lay))))
    with pytest.raises(RuntimeError, match="record fields"):
        rs.DeviceReplayClient(dataclasses.replace(cfg, LEARNER_DEVICE="cuda:0"), conn, timeout=1.0)


def test_the_redis_server_sends_reference_format_stacks_from_strips(rs, monkeypatch):
    """ReplayServer's pickled BATCH keeps the reference's (B, T, 4, 84, 84) `s`, materialised from stored strips."""
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200 import replay as R
    T, B, n = 6, 3, 10
    cfg = r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=2, FRAME_STRIP=True, LEARNER_DEVICE="cpu")
    strips = torch.from_numpy(_strips(n, T, 4))
    draws = []

    class _Table:
        def __len__(self):
            return n

        def sample(self, k, beta=0.4):
            idx = torch.from_numpy(np.random.default_rng(len(draws)).integers(0, n, k))
            draws.append(idx)
            return idx, None, torch.linspace(0.1, 1.0, k)

        def gather(self, idx):
            k = idx.numel()
            return {"state": strips[idx], "action": torch.zeros(k, T, dtype=torch.int32),
                    "reward": torch.zeros(k, T), "h0": torch.zeros(k, 512), "h1": torch.zeros(k, 512),
                    "notdone": torch.ones(k)}

    class _Ingest:
        def __init__(self, cfg, connect=None):
            self.store = _Table()
    monkeypatch.setitem(rs.KINDS, "r2d2", dataclasses.replace(rs.KINDS["r2d2"], replay=_Ingest))
    conn = FakeRedis()
    srv = rs.ReplayServer(cfg, conn)
    assert srv.buffer() == 8
    for k, blob in enumerate(conn.lrange("BATCH", 0, -1)):
        (h0, h1), s, *_ = pickle.loads(blob)
        ii = draws[0][k * B:(k + 1) * B]
        assert isinstance(s, np.ndarray) and s.shape == (B, T, 4, 84, 84) and s.flags.c_contiguous
        np.testing.assert_array_equal(s, _stacks(strips[ii].numpy()))
    assert rs.KINDS["r2d2"].fields(cfg) == R.r2d2_fields(T, strip=True)
    got = rs.KINDS["r2d2"].batch({"state": strips[:B], "action": 0, "reward": 0, "notdone": 0,
                                  "h0": torch.zeros(B, 512), "h1": torch.zeros(B, 512)}, "w", "i")
    assert got[1].shape == (B, T, 4, 84, 84) and got[1].data_ptr() == strips.data_ptr()   # the client's stack view


def test_the_reference_actor_sends_sequences_that_slide(golden):
    """tests/golden/r2d2_actor.npz: the records R2D2/Player.py pushed for two episodes of a stub env whose frames are
    constant-valued (a half-overlap cut and a `done` record per episode).  Every record slides and survives strip
    encoding, through the record decoder as through push_arrays."""
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200 import wire
    g = golden("r2d2_actor")
    values, done = g["values"], g["done"]
    assert values.shape[1:] == (80, 4) and values.shape[0] >= 3
    assert (~done).any() and done.any()                             # both get_traj branches
    stacks = np.broadcast_to(values[:, :, :, None, None], values.shape + (84, 84)).copy()
    for v in values:
        np.testing.assert_array_equal(v[1:, :3], v[:-1, 1:])        # s[t+1][:3] == s[t][1:]
    strips = R.encode_strips(stacks)
    np.testing.assert_array_equal(R.strip_stacks(torch.from_numpy(strips)).numpy(), stacks)
    cols, _ = wire.decode_r2d2([pickle.loads(b) for b in _records(stacks)], 80, strip=True)
    np.testing.assert_array_equal(cols[0], strips)


def test_conv1_refuses_bad_frame_sources_before_any_launch(rs):
    """conv_1's forward and weight gradient refuse a bad frame source, strided or plane table, before any launch."""
    from distributed_rl_b200 import _lib
    lib = _lib.load()
    A = 0x10000                                                     # 16-byte aligned, never dereferenced
    fwd = lambda src: lib.b2rl_conv1_fused(src, None, 8, A, A, 1, 32, A, 0, None)
    bwd = lambda src: lib.b2rl_conv1_wgrad(src, None, 8, A, None, 32, A, A, 0, None)
    strided = [(dict(base=f, table=t, row_stride=stride), msg)
               for f, t, stride, msg in ((A, None, 0, b"row stride"), (A, None, -7056, b"row stride"),
                                         (A, None, 7000, b"row stride"), (A + 8, None, 7056, b"aligned"),
                                         (None, A + 4, 7056, b"aligned"), (None, None, 7056, b"exactly one"),
                                         (A, A, 7056, b"exactly one"))]
    planes = [(dict(pool=A, planes=A, plane_base=2), b"plane_base"), (dict(pool=A + 8, planes=A), b"16-byte aligned"),
              (dict(pool=A, planes=A + 2, plane_base=4), b"4-byte aligned"), (dict(pool=A), b"plane table"),
              (dict(pool=A, planes=A, base=A), b"exactly one"), (dict(pool=A, planes=A, rows=0), b"rows")]
    for call in (fwd, bwd):
        for kw, msg in strided + planes:
            assert call(_lib.Frames(**{"rows": 8, **kw})) < 0, kw
            assert msg in lib.b2rl_last_error(), lib.b2rl_last_error()
