"""CPU checks of the captured R2D2 and IMPALA steps on served minibatches (SERVED_FUSED_STEP): the order in which the
learners' served loops bind a slot, step, release it and write back, over a Redis stand-in with real list semantics
(device work replaced by a log, as test_served_fused_cpu.py does for Ape-X); the refusals, which come before the
learner builds anything; and the frame-row check of ServeRing.bind for records holding several frame stacks."""
import pickle
from types import SimpleNamespace

import pytest
import torch

from fake_redis import FakeRedis
from test_served_fused_cpu import _client


@pytest.fixture(scope="module")
def rs():
    from distributed_rl_b200 import build
    build.build()
    from distributed_rl_b200 import replay_server
    return replay_server


def _step(log, conn, rs, B):
    """A bound step logged with the RELEASE_SLOT count at the time it is enqueued; like a graph replay it returns
    the same output buffers every time, with new values."""
    prio = torch.arange(B, dtype=torch.float32)

    def bound_step():
        log.append(("step", conn.llen(rs.RELEASE_SLOT)))
        prio.add_(1.0)
        return {"scalars": torch.zeros(2), "p_norm": torch.zeros(()), "prio": prio, "idx": torch.arange(B) + 10}
    return bound_step


def _r2d2_learner(client, log, conn, rs, B=4):
    from distributed_rl_b200 import r2d2
    L = object.__new__(r2d2.Learner)
    L.cfg, L._served = r2d2.R2D2Config(BATCHSIZE=B, SERVED_FUSED_STEP=True), True
    L.memory, L._step_state = client, SimpleNamespace(cur={}, frames={})
    L._bound_step = _step(log, conn, rs, B)
    return L


def _impala_learner(client, log, conn, rs, B=4):
    from distributed_rl_b200 import impala
    L = object.__new__(impala.Learner)
    L.cfg, L._served = impala.ImpalaConfig(BATCHSIZE=B, SERVED_FUSED_STEP=True), True
    L._memory, L._bound = client, SimpleNamespace(cur={}, frames={})
    L._bound_step = _step(log, conn, rs, B)
    return L


def test_r2d2_releases_after_the_step_and_the_eviction_step_skips_its_write_back(rs):
    conn, log = FakeRedis(), []
    srv = rs.ServerSlots(conn, 2, 4)
    srv.fill_free(lambda k, seq: None)
    c = _client(rs, conn, log)
    L = _r2d2_learner(c, log, conn, rs)
    tot = L._next_step(1, 2)
    assert tot is not None and tot.shape == (2,)
    # filled[0] is waited on before the bind; the step runs while slot 0 is held; released[0] is recorded behind
    # the step and RELEASE_SLOT hands the slot back; then the write-back goes to update slot 0
    assert log == [("wait", "filled0"), ("bind", 1000), ("step", 0), ("record", "released0"),
                   ("wait", "applied0"), ("put_update", 0, 1, [10, 11, 12, 13], [1.0, 2.0, 3.0, 4.0]),
                   ("record", "written0")]
    assert [pickle.loads(d) for d in conn.lrange(rs.RELEASE_SLOT, 0, -1)] == [(0, 1)]
    del log[:]
    assert L._next_step(2, 2) is not None                  # step 2 % log_every == 0: the eviction request
    assert log == [("wait", "filled1"), ("bind", 2000), ("step", 1), ("record", "released1")]
    assert conn.llen(rs.UPDATE_SLOT) == 1                   # no write-back for this step
    assert c.lock is True
    del log[:]
    assert L._next_step(3, 2) is None                       # nothing filled: no bind, no step, no write-back
    assert ("step", 2) not in log and all(e[0] not in ("bind", "put_update") for e in log)
    assert pickle.loads(conn.get("FLAG_REMOVE")) is True and c.lock is False
    assert srv.collect_releases(lambda k: None) == 2 and sorted(srv.free) == [0, 1]


def test_impala_releases_after_the_step_and_writes_nothing_back(rs):
    conn, log = FakeRedis(), []
    rs.ServerSlots(conn, 2, 4).fill_free(lambda k, seq: None)
    c = _client(rs, conn, log)
    L = _impala_learner(c, log, conn, rs)
    assert L._next_step(0) is True
    assert L._next_step(1) is True
    assert log == [("wait", "filled0"), ("bind", 1000), ("step", 0), ("record", "released0"),
                   ("wait", "filled1"), ("bind", 2000), ("step", 1), ("record", "released1")]
    assert [pickle.loads(d) for d in conn.lrange(rs.RELEASE_SLOT, 0, -1)] == [(0, 1), (1, 2)]
    assert conn.llen(rs.UPDATE_SLOT) == 0
    del log[:]
    assert L._next_step(2) is False                         # nothing filled: run() retries, the step is not counted
    assert all(e[0] not in ("bind", "step") for e in log)


def test_refusals_come_before_anything_is_built(monkeypatch):
    from distributed_rl_b200 import impala, r2d2, replay as R
    built = []
    monkeypatch.setattr(r2d2, "GraphAgent", lambda *a, **k: built.append(1))
    monkeypatch.setattr(impala, "GraphAgent", lambda *a, **k: built.append(1))

    def mem(B, fields):
        fb = [f.nbytes for f in fields]
        return SimpleNamespace(acquire=None, release=None,
                               ring=SimpleNamespace(layout=SimpleNamespace(batch=B, n_fields=len(fb), field_bytes=fb)))
    r2 = dict(BATCHSIZE=8, FIXED_TRAJECTORY=80, SERVED_FUSED_STEP=True, LEARNER_DEVICE="cpu")
    im = dict(BATCHSIZE=8, UNROLL_STEP=20, SERVED_FUSED_STEP=True, LEARNER_DEVICE="cpu")
    cases = ((r2d2.Learner, r2d2.R2D2Config, r2, R.r2d2_fields(80), R.r2d2_fields(40)),
             (impala.Learner, impala.ImpalaConfig, im, R.impala_fields(20), R.impala_fields(10)))
    for Learner, Config, kw, fields, other in cases:
        with pytest.raises(ValueError, match="FUSED_CONV1"):
            Learner(Config(**dict(kw, FUSED_CONV1=False)), memory=mem(8, fields))
        with pytest.raises(TypeError, match="binds ring slots"):
            Learner(Config(**kw), memory=SimpleNamespace(sample=None))
        with pytest.raises(ValueError, match="BATCHSIZE = 8"):
            Learner(Config(**kw), memory=mem(16, fields))
        with pytest.raises(ValueError, match="record fields"):
            Learner(Config(**kw), memory=mem(8, other))
    assert not built


@pytest.mark.parametrize("kind", ["apex", "r2d2", "impala"])
def test_bind_frame_rows_cover_every_frame_stack_of_the_slot(rs, kind):
    """Ape-X: one frame stack per record; R2D2: T per sequence; IMPALA: T + 1 per rollout."""
    from distributed_rl_b200 import replay as R
    B = 4
    fields, stacks = {"apex": (R.APEX_FIELDS, 1), "r2d2": (R.r2d2_fields(80), 80),
                      "impala": (R.impala_fields(20), 21)}[kind]
    table = torch.zeros(2, dtype=torch.int64)
    _, to = rs.bind_targets(B, fields, {}, {"state": R.BoundFrames(table, 1, B * stacks)})
    assert to[0] == table.data_ptr() + 8 and all(to[i] is None for i in range(1, len(fields)))
    for rows in (B, B * stacks - 1, B * stacks + 1):
        if rows == B * stacks:
            continue
        with pytest.raises(ValueError, match=f"{stacks:g} frame stacks per record"):
            rs.bind_targets(B, fields, {}, {"state": R.BoundFrames(table, 1, rows)})
    if kind != "apex":     # a copied field keeps its exact size check
        with pytest.raises(AssertionError, match="action"):
            rs.bind_targets(B, fields, {"action": torch.empty(B, dtype=torch.int32)}, {})
