"""Drop-in for R2D2/ReplayServer.py: `ReplayServer()` (no arguments) + `.run()`."""
from distributed_rl_b200.r2d2 import R2D2Config
from distributed_rl_b200.replay_server import ReplayServer as _Server
from APE_X.ReplayMemory import _connect


class ReplayServer(_Server):
    def __init__(self):
        import configuration as C
        cfg = R2D2Config.from_configuration()
        super().__init__(cfg, connect=_connect(cfg.REDIS_SERVER),
                         connect_push=_connect(getattr(C, "REDIS_SERVER_PUSH", cfg.REDIS_SERVER)))
