"""CPU checks of the stand-alone replay mode for R2D2: the serve-ring layout of the R2D2 sequence record, the record
kind the servers and clients take from their config, the R2D2 drop-ins under the reference's names, and the decision
on the reference's server-mode quirks (DESIGN.md §2): each minibatch is pushed to `BATCH` once, batch-major, and
unpickled once by the consumer."""
import dataclasses
import json
import os
import pickle
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from fake_redis import FakeRedis

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rs():
    from distributed_rl_b200 import build
    build.build()
    from distributed_rl_b200 import replay_server
    return replay_server


def _align(x, a):
    return (x + a - 1) // a * a


@pytest.mark.parametrize("batch", [32, 64])
def test_layout_of_the_r2d2_record(rs, batch):
    """state (80, 4, 84, 84) uint8, action int32[80], reward fp32[80] (the 320-byte rows), h0 / h1 fp32[512],
    notdone fp32: packed in record order after the header, idx and w."""
    from distributed_rl_b200 import replay as R
    fields = R.r2d2_fields(80)
    fb = [f.nbytes for f in fields]
    assert fb == [80 * 28224, 320, 320, 2048, 2048, 4]
    L = rs.serve_layout(batch, 4, fb)
    assert L.idx_off == 16 and L.w_off == 16 + 8 * batch
    off = _align(L.w_off + 4 * batch, 16)
    want = []
    for b in fb:
        want.append(off)
        off = _align(off + b * batch, 16)
    assert [L.field_off[i] for i in range(len(fb))] == want
    assert L.field_off[2] - L.field_off[1] == 320 * batch            # action rows, then reward rows
    assert L.field_off[1] == L.field_off[0] + batch * 2_257_920
    assert L.slot_bytes == _align(want[-1] + 4 * batch, 128)
    if batch == 64:
        assert L.slot_bytes == 144_811_136                           # one B = 64 sequence minibatch: 144.8 MB


def test_the_record_kind_comes_from_the_config(rs):
    from distributed_rl_b200 import apex, r2d2
    from distributed_rl_b200 import replay as R
    ka, kr = rs.record_kind(apex.ApexConfig()), rs.record_kind(r2d2.R2D2Config(FIXED_TRAJECTORY=40))
    assert (ka.replay, ka.m, ka.enough) == (apex.Replay, 32, 32)
    assert (kr.replay, kr.m, kr.enough) == (r2d2.Replay, 8, 18)
    assert ka.fields(apex.ApexConfig()) == R.APEX_FIELDS
    assert kr.fields(r2d2.R2D2Config(FIXED_TRAJECTORY=40)) == R.r2d2_fields(40)
    b = {"state": "s", "next_state": "ns", "action": "a", "reward": "r", "done": "d"}
    assert ka.batch(b, "w", "i") == ["s", "a", "r", "ns", "d", "w", "i"]


def test_a_payload_pool_store_is_refused(rs):
    from distributed_rl_b200 import r2d2
    with pytest.raises(ValueError, match="PAYLOAD_POOL"):
        rs.ReplayServer(r2d2.R2D2Config(PAYLOAD_POOL=16, LEARNER_DEVICE="cpu"), FakeRedis())


class _Store:
    """A CPU stand-in for DeviceReplay: sample() hands out fixed indices, gather() indexes a table."""

    def __init__(self, fields, n, rng):
        import torch
        self.table = {}
        for f in fields:
            shape = (n,) + tuple(f.shape)
            if f.dtype == torch.uint8:
                self.table[f.name] = torch.from_numpy(rng.integers(0, 256, shape, dtype=np.uint8))
            elif f.dtype == torch.int32:
                self.table[f.name] = torch.from_numpy(rng.integers(0, 6, shape).astype(np.int32))
            else:
                self.table[f.name] = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
        self.n = n
        self.draws = []

    def __len__(self):
        return self.n

    def sample(self, k, beta=0.4):
        import torch
        idx = torch.from_numpy(np.random.default_rng(len(self.draws)).integers(0, self.n, k))
        self.draws.append(idx)
        return idx, None, torch.linspace(0.1, 1.0, k)

    def gather(self, idx):
        return {name: t[idx] for name, t in self.table.items()}


def test_the_redis_server_pushes_each_minibatch_once_batch_major_and_the_consumer_decodes_it_once(rs, monkeypatch):
    import torch
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200 import replay as R
    T, B = 8, 3
    cfg = r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=2, LEARNER_DEVICE="cpu")
    store = _Store(R.r2d2_fields(T), 20, np.random.default_rng(0))

    class _Ingest:
        def __init__(self, cfg, connect=None):
            self.store = store
    monkeypatch.setitem(rs.KINDS, "r2d2", dataclasses.replace(rs.KINDS["r2d2"], replay=_Ingest))
    conn = FakeRedis()
    srv = rs.ReplayServer(cfg, conn)
    assert srv.m == 8                                               # R2D2/ReplayServer.py:66
    assert srv.buffer() == 8
    assert conn.llen("BATCH") == 8                                  # once per minibatch, not twice
    idx = store.draws[0]
    for k, blob in enumerate(conn.lrange("BATCH", 0, -1)):
        (h0, h1), s, a, r, nd, w, i = pickle.loads(blob)
        ii = idx[k * B:(k + 1) * B]
        assert torch.equal(i, ii)
        assert s.shape == (B, T, 4, 84, 84)                         # batch-major: sequence b is s[b]
        np.testing.assert_array_equal(s, store.table["state"][ii].numpy())
        np.testing.assert_array_equal(a, store.table["action"][ii].numpy())
        np.testing.assert_array_equal(r, store.table["reward"][ii].numpy())
        np.testing.assert_array_equal(nd, store.table["notdone"][ii].numpy())
        assert torch.is_tensor(h0) and h0.shape == (1, B, 512)      # as r2d2.Replay.buffer builds it
        assert torch.equal(h0[0], store.table["h0"][ii]) and torch.equal(h1[0], store.table["h1"][ii])
        assert torch.equal(w, torch.linspace(0.1, 1.0, 8 * B)[k * B:(k + 1) * B])

    cli = rs.Replay_Server(cfg, conn, conn)
    cli.poll_once()
    assert len(cli.deque) == 8 and conn.llen("BATCH") == 0          # one queued entry per blob
    assert pickle.loads(conn.get("FLAG_ENOUGH")) is False
    got = [cli.sample() for _ in range(8)]
    assert cli.sample() is False
    for k, b in enumerate(got):                                     # each decoded once, in push order
        assert torch.equal(b[6], idx[k * B:(k + 1) * B])
    for _ in range(3):
        srv.buffer()
    cli.poll_once()
    assert len(cli.deque) == 24 and pickle.loads(conn.get("FLAG_ENOUGH")) is True   # > 18 (R2D2/ReplayMemory.py:249)
    cli.update(idx[:B], torch.ones(B))
    assert cli.idx == idx[:B].tolist()


def test_r2d2_dropins_resolve_to_the_stand_alone_replay_classes(tmp_path):
    from distributed_rl_b200.r2d2 import default_r2d2_model
    cfg = {"ALG": "R2D2", "REDIS_SERVER": "localhost", "REDIS_SERVER_PUSH": "localhost", "ACTION_SIZE": 6,
           "ALPHA": 0.9, "BETA": 0.4, "GAMMA": 0.997, "TARGET_FREQUENCY": 2500, "N": 8, "BATCHSIZE": 32,
           "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0", "REPLAY_MEMORY_LEN": 10000, "BUFFER_SIZE": 1000,
           "UNROLL_STEP": 5, "FIXED_TRAJECTORY": 80, "MEM": 20, "USE_RESCALING": True,
           "optim": {"name": "adam", "lr": 1e-4, "eps": 0.001}, "model": default_r2d2_model()}
    (tmp_path / "cfg").mkdir()
    (tmp_path / "cfg" / "ape_x.json").write_text(json.dumps(cfg))
    code = """
        import configuration as C
        assert C.ALG == "R2D2" and C.REDIS_SERVER_PUSH == "localhost"
        from R2D2.ReplayServer import ReplayServer
        from R2D2.ReplayMemory import Replay, Replay_Server
        from R2D2.Learner import Replay_Server as LearnerReplayServer
        import distributed_rl_b200.replay_server as RS
        import distributed_rl_b200.r2d2 as R2
        assert Replay_Server is not Replay and LearnerReplayServer is Replay_Server
        assert issubclass(ReplayServer, RS.ReplayServer) and issubclass(Replay_Server, RS.Replay_Server)
        assert Replay is R2.Replay
        for m in ("update", "buffer", "run"):                  # R2D2/ReplayServer.py
            assert hasattr(ReplayServer, m), m
        for m in ("update", "run", "sample", "start"):         # R2D2/ReplayMemory.py:187-274
            assert hasattr(Replay_Server, m), m
        import inspect
        assert not [p for p in inspect.signature(ReplayServer).parameters]
        assert not [p for p in inspect.signature(Replay_Server).parameters]
        print("OK")
    """
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(REPO, "dropin"), REPO]))
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=tmp_path, env=env, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "OK" in r.stdout
