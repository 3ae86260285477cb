"""Stand-alone replay mode (SURVEY.md §8 f4): `ReplayServer` (APE_X/ReplayServer.py:20-160) owns the prioritized
replay in ITS OWN process / GPU and serves pre-assembled minibatches over the reference's Redis protocol;
`Replay_Server` (APE_X/ReplayMemory.py:170-257) is the learner-side consumer with the `Replay` surface
(`sample()`, `update()`, `start()`).

Keys (the reference's): list `experience` (actors -> server), list `BATCH` on the push connection (server ->
learner: pickled `[s, a, r, s', done, w, idx]`), list `update` (learner -> server: pickled `(idx list, priorities)`),
flags `FLAG_BATCH` (enough data to serve), `FLAG_ENOUGH` (learner has > 32 batches queued), `FLAG_REMOVE` (learner asks
for `remove_to_fit`).

What is GPU-native here is the server's store: sampling, IS weights, gather and priority write-back are the HBM
kernels of libb2rl (one sample launch + one TMA gather per served group of minibatches, applied updates in stream
order); the transport stays the reference's pickled Redis lists — this mode exists so that a deployment which
runs the reference's replay out of process keeps working, not as the fast path (the in-process `Replay` is).
Lists are drained atomically (`wire.drain`), see wire.py."""
from __future__ import annotations

import pickle
import threading
import time

import numpy as np
import torch

from . import wire
from .apex import ApexConfig
from .learner_common import Stoppable


class ReplayServer(Stoppable):
    def __init__(self, cfg: ApexConfig | None = None, connect=None, connect_push=None, m: int = 32):
        super().__init__()
        self.cfg = cfg or ApexConfig.from_configuration()
        self.device = torch.device(self.cfg.LEARNER_DEVICE)
        from .apex import Replay
        self._ingest = Replay(self.cfg, connect=None)      # never started: its record decoder + pinned staging + store
        self.store = self._ingest.store
        self.connect, self.connect_push = connect, connect_push if connect_push is not None else connect
        self.m = m                               # minibatches assembled per buffer() (the reference: 32, :66)
        self.FLAG_BATCH = self.FLAG_REMOVE = False
        self.total_transition = 0
        if self.connect is not None:
            self.connect.set("FLAG_BATCH", pickle.dumps(False))           # :39

    def update(self) -> int:
        """:41-63 — apply the learner's queued priority write-backs."""
        data = wire.drain(self.connect, "update")
        if not data:
            return 0
        idx_list, vals_list = [], []
        for d in data:
            idx, vals = pickle.loads(d)
            idx_list += [int(i) for i in idx]
            vals_list.append(np.asarray(vals, np.float32))
        self.store.update(torch.as_tensor(np.asarray(idx_list, np.int64)).to(self.device),
                          torch.as_tensor(np.concatenate(vals_list, 0)).to(self.device))
        return len(idx_list)

    def buffer(self) -> int:
        """:65-114 — sample BATCHSIZE * m, IS weights, assemble m minibatches, RPUSH them to `BATCH`."""
        B, m = self.cfg.BATCHSIZE, self.m
        idx, _, w = self.store.sample(B * m, beta=self.cfg.BETA)
        b = self.store.gather(idx)
        s, ns = b["state"].cpu().numpy(), b["next_state"].cpu().numpy()
        a, r, d = b["action"].cpu().numpy(), b["reward"].cpu().numpy(), b["done"].cpu().numpy().astype(bool)
        w, idx = w.cpu(), idx.cpu()
        blobs = []
        for k in range(m):
            sl = slice(k * B, (k + 1) * B)
            blobs.append(pickle.dumps([s[sl], a[sl], r[sl], ns[sl], d[sl], w[sl], idx[sl]]))
        return self.connect_push.rpush("BATCH", *blobs)

    def serve_once(self) -> dict:
        """One iteration of run() (:116-160)."""
        k = self.cfg.BUFFER_SIZE
        if len(self.store) > k and not self.FLAG_BATCH:
            self.FLAG_BATCH = True
            self.connect.set("FLAG_BATCH", pickle.dumps(True))
        data = wire.drain(self.connect, "experience")
        pushed = 0
        if data:
            self._ingest.push_records(data)
            self.total_transition += len(data)
            if len(self.store) > k:
                pushed = self.buffer()
        applied = self.update()
        if len(self.store) >= self.cfg.REPLAY_MEMORY_LEN:
            cond = self.connect.get("FLAG_REMOVE")
            if cond is not None and pickle.loads(cond):
                over = len(self.store) - self.cfg.REPLAY_MEMORY_LEN
                if over > 0:
                    self.store.evict(over)
                self.connect.set("FLAG_REMOVE", pickle.dumps(False))
        return {"ingested": len(data), "batches_queued": pushed, "updates_applied": applied}

    def run(self):
        while not self._stop_evt.is_set():
            st = self.serve_once()
            if st["batches_queued"] > 100:
                time.sleep(1)                   # the learner is behind: :143-144
            elif not st["ingested"]:
                time.sleep(0.002)


class Replay_Server(Stoppable, threading.Thread):
    """Learner-side consumer of a ReplayServer: same surface as `Replay` (sample / update / start / lock)."""

    def __init__(self, cfg: ApexConfig | None = None, connect=None, connect_push=None):
        super().__init__(daemon=True)
        self.cfg = cfg or ApexConfig.from_configuration()
        self.connect, self.connect_push = connect, connect_push if connect_push is not None else connect
        self._lock = threading.Lock()
        self.deque, self.idx, self.vals = [], [], []
        self.lock = False

    def update(self, idx, vals) -> None:
        """:188-190 — queue; flushed to the server's `update` list beyond 1000 entries."""
        with self._lock:
            self.idx += [int(i) for i in idx]
            self.vals.append(np.asarray(vals.detach().cpu() if torch.is_tensor(vals) else vals, np.float32))

    def poll_once(self) -> None:
        data = wire.drain(self.connect_push, "BATCH")
        if data:
            with self._lock:
                self.deque += data
        self.connect.set("FLAG_ENOUGH", pickle.dumps(len(self.deque) > 32))       # :232-239
        if self.lock:                                                              # eviction request -> the server's flag
            self.connect.set("FLAG_REMOVE", pickle.dumps(True))
            self.lock = False
        with self._lock:
            if len(self.idx) > 1000:                                               # :241-249
                self.connect.rpush("update", pickle.dumps((self.idx[:], np.concatenate(self.vals, 0))))
                self.idx.clear(); self.vals.clear()

    def run(self):
        while not self._stop_evt.is_set():
            self.poll_once()
            time.sleep(0.001)

    def sample(self):
        with self._lock:
            if not self.deque:
                return False
            blob = self.deque.pop(0)
        return pickle.loads(blob)
