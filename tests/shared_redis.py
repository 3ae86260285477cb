"""The Redis stand-in of tests/fake_redis.py shared between processes: hosted by a multiprocessing manager, with a
redis-py shim whose pipelines are built locally and executed atomically in the manager.  Used by the two-process
serve tests and by tools/bench_serve.py (the GPU hosts run no Redis server).  Test infrastructure only."""
from multiprocessing.managers import BaseManager

from fake_redis import FakeRedis


class SharedRedis(FakeRedis):
    """FakeRedis hosted by a manager: a pipeline arrives as one list of commands and runs under the lock."""

    def run_pipeline(self, cmds):
        with self._mu:
            return [getattr(self, "_" + name)(*a) for name, a in cmds]


class RedisManager(BaseManager):
    pass


RedisManager.register("Redis", SharedRedis)


class _Pipe:
    def __init__(self, proxy):
        self._p, self._cmds = proxy, []

    def __getattr__(self, name):
        def queue(*a):
            self._cmds.append((name, a))
            return self
        return queue

    def execute(self):
        cmds, self._cmds = self._cmds, []
        return self._p.run_pipeline(cmds)


class Shim:
    """redis-py surface over the manager proxy (picklable: hand it to a `spawn` child as is)."""

    def __init__(self, proxy):
        self._p = proxy

    def pipeline(self):
        return _Pipe(self._p)

    def __getattr__(self, name):
        if name.startswith("__") or name == "_p":
            raise AttributeError(name)
        return getattr(self._p, name)
