"""CPU checks of the served fused Ape-X step (ApexConfig.SERVED_FUSED_STEP): the order in which
DeviceReplayClient.acquire / release and the learner's step enqueue their work and post their descriptors, over a
Redis stand-in with real list semantics (device work replaced by a log), and the refusals of the learner and of the
new C entry points, which reject bad arguments before any CUDA call."""
import ctypes
import pickle
from collections import deque
from types import SimpleNamespace

import pytest
import torch

from fake_redis import FakeRedis


@pytest.fixture(scope="module")
def rs():
    from distributed_rl_b200 import build
    build.build()
    from distributed_rl_b200 import replay_server
    return replay_server


class _Ev:
    def __init__(self, log, name):
        self.log, self.name = log, name

    def record(self, stream):
        self.log.append(("record", self.name))


class _Stream:
    def __init__(self, log):
        self.log = log

    def wait_event(self, ev):
        self.log.append(("wait", ev.name))


class _Ring:
    """The client's ring with the device work logged: slot k of the mapped ring starts at 1000 * (k + 1)."""

    def __init__(self, log, batch, slots):
        self.log = log
        self.layout = SimpleNamespace(batch=batch, slots=slots, slot_bytes=4096)

    def slot_ptrs(self, k):
        return [1000 * (k + 1)], None

    def bind(self, base, fields, out, frames, stream):
        self.log.append(("bind", base))

    def take(self, k, dst, stream):
        self.log.append(("take", k))

    def put_update(self, j, seq, idx, prio, stream):
        self.log.append(("put_update", j, seq, idx.tolist(), prio.tolist()))


def _client(rs, conn, log, B=4, slots=2, same_gpu=True):
    from distributed_rl_b200 import apex, replay as R
    c = object.__new__(rs.DeviceReplayClient)
    c.cfg, c.kind, c.fields = apex.ApexConfig(BATCHSIZE=B), rs.KINDS["apex"], R.APEX_FIELDS
    c.device = torch.device("cpu")
    c.server_device = c.device if same_gpu else torch.device("meta")
    c.connect, c.lock, c.ring = conn, False, _Ring(log, B, slots)
    c.filled, c.released, c.applied, c.written = ([_Ev(log, f"{n}{k}") for k in range(slots)]
                                                  for n in ("filled", "released", "applied", "written"))
    c.slots = rs.ClientSlots(conn, slots)
    c._pending, c._held, c._stage, c.last_served = deque(), None, None, None
    stream = _Stream(log)
    c._stream = lambda: stream
    return c


def _learner(client, log, conn, rs, B=4):
    """An apex.Learner reduced to what _next_step touches on a served memory; its step is logged with the RELEASE_SLOT
    count at the time the step is enqueued."""
    from distributed_rl_b200 import apex
    L = object.__new__(apex.Learner)
    L.cfg, L._served = apex.ApexConfig(BATCHSIZE=B, SERVED_FUSED_STEP=True), True
    L.memory, L._fused = client, SimpleNamespace(cur={}, frames={})
    prio = torch.arange(B, dtype=torch.float32)

    def fused_step():
        log.append(("step", conn.llen(rs.RELEASE_SLOT)))
        prio.add_(1.0)                     # like a graph replay: the same output buffer, new values
        return {"scalars": torch.zeros(3), "p_norm": torch.zeros(()), "prio": prio, "idx": torch.arange(B) + 10}
    L.fused_step = fused_step
    return L


def test_the_slot_is_released_after_the_step_and_the_eviction_step_skips_its_write_back(rs):
    conn, log = FakeRedis(), []
    srv = rs.ServerSlots(conn, 2, 4)
    srv.fill_free(lambda k, seq: None)
    c = _client(rs, conn, log)
    L = _learner(c, log, conn, rs)
    assert L._next_step(1, 2) is not None
    # filled[0] is waited on before the bind; the step runs while slot 0 is still held; released[0] is recorded
    # behind the step, then RELEASE_SLOT hands the slot back; then the write-back goes to update slot 0
    assert log == [("wait", "filled0"), ("bind", 1000), ("step", 0), ("record", "released0"),
                   ("wait", "applied0"), ("put_update", 0, 1, [10, 11, 12, 13], [1.0, 2.0, 3.0, 4.0]),
                   ("record", "written0")]
    assert [pickle.loads(d) for d in conn.lrange(rs.RELEASE_SLOT, 0, -1)] == [(0, 1)]
    assert conn.llen(rs.UPDATE_SLOT) == 1
    del log[:]
    assert L._next_step(2, 2) is not None                  # step 2 % log_every == 0: the eviction request
    assert log == [("wait", "filled1"), ("bind", 2000), ("step", 1), ("record", "released1")]
    assert conn.llen(rs.UPDATE_SLOT) == 1                   # no write-back for this step
    assert c.lock is True and conn.get("FLAG_REMOVE") is None
    assert [pickle.loads(d) for d in conn.lrange(rs.RELEASE_SLOT, 0, -1)] == [(0, 1), (1, 2)]
    assert L._next_step(3, 2) is None                       # nothing filled; the poll raised the server's flag
    assert pickle.loads(conn.get("FLAG_REMOVE")) is True and c.lock is False
    assert srv.collect_releases(lambda k: None) == 2 and sorted(srv.free) == [0, 1]


def test_a_slot_from_another_gpu_is_staged_and_released_before_the_step(rs):
    conn, log = FakeRedis(), []
    rs.ServerSlots(conn, 2, 4).fill_free(lambda k, seq: None)
    c = _client(rs, conn, log, same_gpu=False)
    c._stage = torch.empty(8, dtype=torch.uint8)           # the persistent local copy (allocated on first use)
    L = _learner(c, log, conn, rs)
    L._next_step(1, 100)
    stage = c._stage.data_ptr()
    assert log[:5] == [("wait", "filled0"), ("take", 0), ("record", "released0"), ("bind", stage), ("step", 1)]
    c2 = c._stage
    L._next_step(2, 100)
    assert c._stage is c2                                   # one buffer for every step
    assert [pickle.loads(d) for d in conn.lrange(rs.RELEASE_SLOT, 0, -1)] == [(0, 1), (1, 2)]


def test_queued_write_backs_own_their_data(rs):
    """With every update slot with the server, update() queues the write-back; a graph's static outputs are
    overwritten by the next replay, so what is queued must be a copy."""
    conn, log = FakeRedis(), []
    c = _client(rs, conn, log, slots=1)
    idx, prio = torch.arange(4), torch.full((4,), 0.5)
    c.update(idx, prio)                                     # takes the only update slot
    c.update(idx, prio)                                     # queued
    c.update(idx, prio)
    assert len(c._pending) == 2
    idx.add_(100)
    prio.fill_(9.0)                                         # the next replay writes its outputs
    assert all(i.tolist() == [0, 1, 2, 3] and v.tolist() == [0.5] * 4 for i, v in c._pending)
    srv = rs.ServerSlots(conn, 1, 4)
    srv.apply_updates(lambda j, n: None)
    c.slots.poll()
    c._flush_updates()
    assert log[-2] == ("put_update", 0, 2, [0, 1, 2, 3], [0.5] * 4)


def test_served_fused_step_refusals(rs):
    from distributed_rl_b200 import apex
    mem = SimpleNamespace(acquire=None, release=None, ring=SimpleNamespace(layout=SimpleNamespace(batch=64)))
    with pytest.raises(ValueError, match="FUSED_CONV1"):
        apex.Learner(apex.ApexConfig(BATCHSIZE=64, FUSED_CONV1=False, SERVED_FUSED_STEP=True,
                                     LEARNER_DEVICE="cpu"), memory=mem)
    with pytest.raises(ValueError, match="BATCHSIZE = 32"):
        apex.Learner(apex.ApexConfig(BATCHSIZE=32, SERVED_FUSED_STEP=True, LEARNER_DEVICE="cpu"), memory=mem)
    with pytest.raises(TypeError, match="binds ring slots"):
        apex.Learner(apex.ApexConfig(BATCHSIZE=64, SERVED_FUSED_STEP=True, LEARNER_DEVICE="cpu"),
                     memory=SimpleNamespace(sample=None, update=None))
    L = object.__new__(apex.Learner)
    L.cfg, L._served = apex.ApexConfig(SERVED_FUSED_STEP=True), True
    with pytest.raises(ValueError, match="data parallelism"):
        L.enable_data_parallel()


def test_serve_bind_and_table_sources_reject_bad_arguments_before_any_launch(rs):
    from distributed_rl_b200 import _lib, replay as R
    lib = _lib.load()
    L = rs.serve_layout(8, 2, [f.nbytes for f in R.APEX_FIELDS])
    bufs = [ctypes.c_void_p(0x10000 * (i + 1)) for i in range(3)]
    fo = (ctypes.c_void_p * _lib.MAX_FIELDS)()
    assert lib.b2rl_serve_bind(None, ctypes.byref(L), 8, *bufs, fo, fo, None) < 0
    assert b"null slot" in lib.b2rl_last_error()
    assert lib.b2rl_serve_bind(0x100008, ctypes.byref(L), 8, *bufs, fo, fo, None) < 0
    assert b"16-byte" in lib.b2rl_last_error()
    assert lib.b2rl_serve_bind(0x100000, ctypes.byref(L), 9, *bufs, fo, fo, None) < 0
    assert b"batch does not match" in lib.b2rl_last_error()
    both = (ctypes.c_void_p * _lib.MAX_FIELDS)(0x20000)
    assert lib.b2rl_serve_bind(0x100000, ctypes.byref(L), 8, *bufs, both, both, None) < 0
    assert b"not both" in lib.b2rl_last_error()
    table = lambda entry: _lib.Frames(table=entry, row_stride=R.FRAME_STACK_BYTES, rows=8)
    assert lib.b2rl_conv1_fused(table(None), None, 8, 0x1000, 0x1000, 1, 32, 0x1000, 1, None) < 0
    assert b"null frame source" in lib.b2rl_last_error()
    assert lib.b2rl_conv1_fused(table(0x1004), None, 8, 0x1000, 0x1000, 1, 32, 0x1000, 1, None) < 0
    assert b"8-byte" in lib.b2rl_last_error()
    assert lib.b2rl_conv1_wgrad(table(None), None, 8, 0x1000, None, 32, 0x1000, 0x1000, 0, None) < 0
    assert b"null frame source" in lib.b2rl_last_error()
