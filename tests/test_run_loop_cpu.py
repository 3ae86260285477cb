"""CPU checks of the Ape-X and R2D2 `Learner.run()` loops: the write-back and eviction cadence (`memory.lock` every
`log_every` steps, that step's write-back skipped, inline eviction only without a running ingest thread), retried
steps when no minibatch is ready, target syncs, parameter snapshots and the logged averages.  The step, the replay
and the publishers are fakes; the Redis stand-in has real list semantics."""
import pickle
import re
from types import SimpleNamespace

import pytest
import torch

from fake_redis import FakeRedis

STEPS, LOG_EVERY, TARGET_FREQUENCY = 100, 20, 30
LOCK_STEPS = [20, 40, 60, 80, 100]
SYNCS = [30, 60, 90]
NONE_CALLS = {3, 4, 22}          # attempts that find no minibatch; the 22nd is the first try of step 20


class _Log:
    """What the fakes saw.  Each entry carries `step`, the number of learner steps run when it happened."""

    def __init__(self, none_calls=NONE_CALLS):
        self.none_calls = set(none_calls)
        self.step = 0
        self.calls = 0           # attempts to get a minibatch
        self.locks, self.evicts, self.thread_evicts, self.flag_removes = [], [], [], []
        self.updates, self.syncs, self.snapshots, self.order = [], [], [], []
        self.polls = 0

    def attempt(self) -> bool:
        """One attempt to get a minibatch: False on the `none_calls` attempts."""
        self.calls += 1
        return self.calls not in self.none_calls

    def ran(self) -> int:
        self.step += 1
        return self.step


@pytest.fixture
def log(monkeypatch):
    """A fresh log, and learner_common.ParamPublisher (which needs CUDA) replaced by a recorder writing to it."""
    from distributed_rl_b200 import learner_common
    lg = _Log()

    class Recorder:
        def __init__(self, model, connect, key, count_key, wrap=None, on_ready=None):
            self.key = key

        def snapshot(self, step):
            lg.snapshots.append((lg.step, self.key, step))

        def poll(self):
            lg.polls += 1

    monkeypatch.setattr(learner_common, "ParamPublisher", Recorder)
    return lg


class _Stats:
    max_weight = 0.5

    def __len__(self):
        return 1000


class _Memory:
    """A replay as run() sees it.  In-process: its ingest thread is alive or not; a live thread serves the eviction
    request before the next minibatch is drawn.  Served: the client's poll, run by sample() / acquire() while the
    request is pending, passes it on to the server and clears it."""

    def __init__(self, log, served, alive=False):
        self.log, self.served, self.alive = log, served, alive
        self.memory = _Stats()
        self._request = False

    @property
    def lock(self):
        return self._request

    @lock.setter
    def lock(self, v):
        if v:
            self.log.locks.append(self.log.step)
        self._request = v

    def is_alive(self):
        return self.alive

    def _evict_on_request(self):
        assert not self.served, "a served memory's server evicts"
        self.log.evicts.append(self.log.step)
        self.lock = False

    def drawn(self):
        """A minibatch is about to be drawn: whatever serves the eviction request has had its turn."""
        if self.lock:
            if self.served:
                self.log.flag_removes.append(self.log.step)
            else:
                assert self.alive, "no thread serves the request of an in-process replay without an ingest thread"
                self.log.thread_evicts.append(self.log.step)
            self.lock = False

    def update(self, idx, prio):
        self.log.updates.append((self.log.step, torch.as_tensor(idx).tolist(), torch.as_tensor(prio).tolist()))
        self.log.order.append("update")

    def sample(self):
        self.drawn()
        return ["batch"] if self.log.attempt() else False

    def acquire(self, cur, frames):
        assert self.served and cur == {} and frames == {}
        self.drawn()
        if not self.log.attempt():
            return None
        self.log.order.append("acquire")
        return (0, self.log.calls, 4)

    def release(self):
        self.log.order.append("release")


class _Net(torch.nn.Linear):
    def __init__(self, log):
        super().__init__(2, 2)
        self.log = log

    def updateParameter(self, model, tau):
        assert tau == 1
        self.log.syncs.append(self.log.step)


class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, value, step):
        self.scalars.append((tag, value, step))


def _stats(n, k):
    """Step n's logged stats: stat i is (i + 1) * n."""
    return torch.tensor([float((i + 1) * n) for i in range(k)])


def _learner(cls, cfg, log, memory, **methods):
    L = object.__new__(cls)
    L.cfg, L.memory, L._served = cfg, memory, memory.served
    L.model, L.target_model = _Net(log), _Net(log)
    L.connect, L.writer = FakeRedis(), _Writer()
    L.connect.rpush("reward", pickle.dumps(1.0), pickle.dumps(3.0))       # drained by the first log
    for name, f in methods.items():
        setattr(L, name, f)
    return L


def _run(L, log, capsys, names, publish_every):
    assert L.run(max_steps=STEPS, log_every=LOG_EVERY) == STEPS
    assert log.step == STEPS and log.calls == STEPS + len(log.none_calls)
    assert pickle.loads(L.connect.get("Start")) is True
    # target sync every TARGET_FREQUENCY steps, with a snapshot of the target's weights at that step; the online
    # weights every `publish_every` steps, snapshot as step - 50
    assert log.syncs == SYNCS
    assert [e for e in log.snapshots if e[1] == "target_state_dict"] == [(s, "target_state_dict", s) for s in SYNCS]
    assert [e for e in log.snapshots if e[1] == "state_dict"] == [
        (s, "state_dict", s - 50) for s in range(publish_every, STEPS + 1, publish_every)]
    assert log.polls == 2 * STEPS             # both publishers, every step
    # every LOG_EVERY steps: the stats averaged over the window
    lines = [re.sub(r"TIME:[0-9.]+", "TIME:*", x) for x in capsys.readouterr().out.splitlines()]
    assert len(lines) == STEPS // LOG_EVERY
    last = sum(range(81, 101)) / 20.0
    want = {name: (i + 1) * last for i, name in enumerate(names)}
    assert set(L.last_log) == {"step", "reward", "time_per_step", *names}
    assert {k: v for k, v in L.last_log.items() if k != "time_per_step"} == dict(want, step=100, reward=-21.0)
    first = sum(range(1, 21)) / 20.0
    mv, norm = (names.index("mean_value") + 1) * first, (names.index("norm") + 1) * first
    assert L.writer.scalars[:3] == [("Reward", 2.0, 20), ("value", mv, 20), ("norm", norm, 20)]
    assert len(L.writer.scalars) == 1 + 2 * len(lines)
    return lines


# ---- Ape-X -----------------------------------------------------------------------------------------------------------
APEX_STATS = ("loss", "mean_value", "mean_weight", "norm")
APEX_LAST = ("step:100 // mean_value:181.000 // norm: 362.000 // REWARD:-21.000 // NUM_MEMORY:1000 // "
             "Mean_Weight:271.500 // MAX_WEIGHT:0.500 // TIME:* // loss:90.50000")


def _apex_cfg(**kw):
    from distributed_rl_b200 import apex
    return apex.ApexConfig(BATCHSIZE=4, BUFFER_SIZE=10, TARGET_FREQUENCY=TARGET_FREQUENCY, LEARNER_DEVICE="cpu", **kw)


@pytest.mark.parametrize("alive", [False, True])
def test_apex_in_process(log, capsys, alive):
    """The in-process step writes its priorities back inside its graph: run() never calls update().  Every LOG_EVERY
    steps it raises the eviction request, which is served inline when no ingest thread runs."""
    from distributed_rl_b200 import apex
    log.none_calls = set()                    # the in-process step always has a minibatch
    mem = _Memory(log, served=False, alive=alive)

    def fused_step():
        mem.drawn()                           # the graph draws from the replay
        assert log.attempt()
        s = _stats(log.ran(), 4)
        return {"scalars": s[:3], "p_norm": s[3], "prio": torch.ones(4), "idx": torch.arange(4)}
    L = _learner(apex.Learner, _apex_cfg(), log, mem, fused_step=fused_step)
    lines = _run(L, log, capsys, APEX_STATS, 50)
    assert log.locks == LOCK_STEPS and log.updates == []
    assert log.evicts == ([] if alive else LOCK_STEPS)
    assert log.thread_evicts == (LOCK_STEPS[:-1] if alive else [])
    assert lines[-1] == APEX_LAST


def test_apex_served(log, capsys):
    """sample() -> train(): every step writes back except every LOG_EVERY-th, which raises the eviction request; the
    client's next poll passes it on.  A step without a minibatch is retried and not counted."""
    from distributed_rl_b200 import apex
    mem = _Memory(log, served=True)

    def train(batch):
        assert batch == ["batch"]
        n = log.ran()
        s = _stats(n, 4)
        return {"loss": s[0], "mean_value": s[1], "p_norm": s[3].reshape(1)}, torch.full((4,), n + 0.5), \
            torch.arange(4) + n, s[2]
    L = _learner(apex.Learner, _apex_cfg(), log, mem, train=train)
    lines = _run(L, log, capsys, APEX_STATS, 50)
    assert log.locks == LOCK_STEPS and log.evicts == [] and log.flag_removes == LOCK_STEPS[:-1]
    assert log.updates == [(n, [n + i for i in range(4)], [n + 0.5] * 4) for n in range(1, STEPS + 1)
                           if n not in LOCK_STEPS]
    assert lines[-1] == APEX_LAST


def test_apex_served_fused(log, capsys):
    """SERVED_FUSED_STEP: acquire() -> the captured step -> release(), then the same write-back cadence.  The step's
    outputs are static buffers that every replay overwrites."""
    from distributed_rl_b200 import apex
    mem = _Memory(log, served=True)
    prio, idx = torch.zeros(4), torch.zeros(4, dtype=torch.int64)

    def fused_step():
        n = log.ran()
        log.order.append("step")
        prio.fill_(n + 0.25)
        idx.copy_(torch.arange(4) + 2 * n)
        s = _stats(n, 4)
        return {"scalars": s[:3], "p_norm": s[3], "prio": prio, "idx": idx}
    L = _learner(apex.Learner, _apex_cfg(SERVED_FUSED_STEP=True), log, mem, fused_step=fused_step)
    L._fused = SimpleNamespace(cur={}, frames={})
    lines = _run(L, log, capsys, APEX_STATS, 50)
    assert log.locks == LOCK_STEPS and log.evicts == [] and log.flag_removes == LOCK_STEPS[:-1]
    assert log.updates == [(n, [2 * n + i for i in range(4)], [n + 0.25] * 4) for n in range(1, STEPS + 1)
                           if n not in LOCK_STEPS]
    want = []
    for n in range(1, STEPS + 1):
        want += ["acquire", "step", "release"] + ([] if n in LOCK_STEPS else ["update"])
    assert log.order == want
    assert lines[-1] == APEX_LAST


# ---- R2D2 ------------------------------------------------------------------------------------------------------------
R2D2_STATS = ("mean_value", "norm")
R2D2_LAST = ("step:100 // mean_value:90.500 // norm: 181.000 // REWARD:-21.000 // NUM_MEMORY:1000 // "
             "MAX_WEIGHT:0.500 // TIME:*")


def _r2d2(log, mem):
    from distributed_rl_b200 import r2d2
    cfg = r2d2.R2D2Config(BATCHSIZE=4, BUFFER_SIZE=10, TARGET_FREQUENCY=TARGET_FREQUENCY, LEARNER_DEVICE="cpu")

    def train(batch):
        assert batch == ["batch"]
        n = log.ran()
        s = _stats(n, 2)
        return {"mean_value": s[0], "p_norm": s[1].reshape(1)}, torch.full((4,), n + 0.75), torch.arange(4) + 3 * n
    return _learner(r2d2.Learner, cfg, log, mem, train=train)


def _r2d2_updates(skipped):
    return [(n, [3 * n + i for i in range(4)], [n + 0.75] * 4) for n in range(1, STEPS + 1) if n not in skipped]


@pytest.mark.parametrize("alive", [False, True])
def test_r2d2_in_process(log, capsys, alive):
    """The eviction request every LOG_EVERY steps.  Without an ingest thread it is served inline, which clears
    `lock`, so that step still writes back; with one, that step's write-back is skipped."""
    L = _r2d2(log, _Memory(log, served=False, alive=alive))
    lines = _run(L, log, capsys, R2D2_STATS, 25)
    assert log.locks == LOCK_STEPS
    assert log.evicts == ([] if alive else LOCK_STEPS)
    assert log.thread_evicts == (LOCK_STEPS[:-1] if alive else [])
    assert log.updates == _r2d2_updates(LOCK_STEPS if alive else ())
    assert lines[-1] == R2D2_LAST


def test_r2d2_served(log, capsys):
    L = _r2d2(log, _Memory(log, served=True))
    lines = _run(L, log, capsys, R2D2_STATS, 25)
    assert log.locks == LOCK_STEPS and log.evicts == [] and log.flag_removes == LOCK_STEPS[:-1]
    assert log.updates == _r2d2_updates(LOCK_STEPS)
    assert lines[-1] == R2D2_LAST
