"""Drop-in for R2D2/ReplayMemory.py: `Replay` and `Replay_Server`, the consumer of a stand-alone R2D2 ReplayServer
(:187-274)."""
from distributed_rl_b200.r2d2 import R2D2Config, Replay  # noqa: F401
from distributed_rl_b200.replay_server import Replay_Server as _ReplayServerClient
from APE_X.ReplayMemory import _connect


class Replay_Server(_ReplayServerClient):
    """Consumer of a stand-alone R2D2 ReplayServer: `BATCH` minibatches in, `update` priorities out."""

    def __init__(self):
        import configuration as C
        cfg = R2D2Config.from_configuration()
        super().__init__(cfg, connect=_connect(cfg.REDIS_SERVER),
                         connect_push=_connect(getattr(C, "REDIS_SERVER_PUSH", cfg.REDIS_SERVER)))
