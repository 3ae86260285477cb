"""Drop-in for R2D2/Learner.py."""
from distributed_rl_b200.r2d2 import R2D2Config, Learner as _Learner  # noqa: F401
from R2D2.ReplayMemory import Replay, Replay_Server  # noqa: F401  (R2D2/Learner.py:5)


class Learner(_Learner):
    def __init__(self):
        from APE_X.ReplayMemory import _connect
        cfg = R2D2Config.from_configuration()
        super().__init__(cfg, connect=_connect(cfg.REDIS_SERVER))
