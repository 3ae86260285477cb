"""CPU model of the frame-deduplicated R2D2 store (R.StripDedupReplay, DESIGN.md §4.18, csrc/dedup.cu with the Strips
layout) and a generator of the sequences the reference R2D2 actors send (R2D2/Player.py).

The model keeps the rule of tests/dedup_model.py, for records of R = T + 3 frames: the 64-bit frame key (frame_keys),
the lowest-position rule inside a batch, the window, the sequence numbers of the misses in batch order, and both
eviction conditions.  The GPU store must give the same pool ids, liveness and priorities for the same stream."""
from __future__ import annotations

import numpy as np

from dedup_model import ALL_KEY_BITS, frame_keys

MAX_FRAMES = 65536          # frames per push: the batch scratch of csrc/dedup.cu


def max_batch(capacity: int, pool_frames: int, window: int, R: int) -> int:
    """Sequences per push (b2rl_dedup_info): larger pushes are split into chunks of this many."""
    return min(capacity, (pool_frames - window - 1) // R, MAX_FRAMES // R)


class StripDedupModel:
    def __init__(self, capacity: int, pool_frames: int, window: int, T: int, mask: int = ALL_KEY_BITS):
        self.cap, self.F, self.W, self.R, self.mask = capacity, pool_frames, window, T + 3, mask
        self.pool = np.zeros((pool_frames, 84, 84), np.uint8)
        self.table = {}                       # key -> seq of the newest frame stored under it
        self.head = 0                         # frames stored so far
        self.slot_head, self.size = 0, 0
        self.ins = np.zeros(capacity, np.int64)
        self.planes = np.zeros((capacity, self.R), np.int32)
        self.prio = np.zeros(capacity, np.float32)
        self.new_frames = []                  # frames stored per pushed chunk

    def push(self, strips: np.ndarray, prio: np.ndarray) -> None:
        mb = max_batch(self.cap, self.F, self.W, self.R)
        for a in range(0, len(prio), mb):
            self._push(strips[a:a + mb], prio[a:a + mb])

    def _push(self, strips, prio):
        n, R = len(prio), self.R
        frames = np.asarray(strips, np.uint8).reshape(R * n, 84, 84)
        keys = frame_keys(frames, self.mask)
        first, seq = {}, np.full(R * n, -1, np.int64)
        rep = np.arange(R * n)
        head = self.head
        for j, k in enumerate(keys.tolist()):
            f = first.setdefault(k, j)
            if f < j and np.array_equal(frames[f], frames[j]):
                rep[j] = f
                continue
            c = self.table.get(k, -1)
            if c >= 0 and c >= head - self.W and np.array_equal(self.pool[c % self.F], frames[j]):
                seq[j] = c
        misses = [j for j in range(R * n) if rep[j] == j and seq[j] < 0]
        for r, j in enumerate(misses):
            seq[j] = head + r
        head_new = head + len(misses)
        # eviction: oldest slots with F - W or more frames stored since their batch began
        tail = (self.slot_head - self.size) % self.cap
        while self.size > 0 and head_new - self.ins[tail] >= self.F - self.W:
            self.prio[tail] = 0.0
            tail = (tail + 1) % self.cap
            self.size -= 1
        for j in misses:
            self.pool[seq[j] % self.F] = frames[j]
            self.table[int(keys[j])] = max(self.table.get(int(keys[j]), -1), int(seq[j]))
        for i in range(n):
            slot = (self.slot_head + i) % self.cap
            self.planes[slot] = seq[rep[R * i:R * i + R]] % self.F
            self.ins[slot] = head
            self.prio[slot] = prio[i]
        self.slot_head = (self.slot_head + n) % self.cap
        self.size = min(self.size + n, self.cap)
        self.head = head_new
        self.new_frames.append(len(misses))

    def live_slots(self) -> np.ndarray:
        return (self.slot_head - self.size + np.arange(self.size)) % self.cap

    def strips(self, slots) -> np.ndarray:
        """The (m, T + 3, 84, 84) strips the pool ids of `slots` name."""
        return self.pool[self.planes[np.asarray(slots)]]


def player_sequences(n: int, T: int = 80, actors: int = 4, episode=(120, 400), seed: int = 0, hidden: int = 512):
    """n sequences as `actors` reference R2D2 actors send them, interleaved as their episodes progress in lock step.

    An episode of E steps (uniform in `episode`) has observations o_0 .. o_E of random frames; its stacks are the last
    four observations, the first one being o_0 four times (R2D2/Player.py:257-267), so stack k is o_max(0, k-3) ..
    o_k.  LocalBuffer.get_traj (:37-62) sends stacks [a, a + T) once the buffer holds int(1.6 T) stacks and then
    drops the first T / 2, and at the episode's end (with its last stack, :306-308) the buffer's last T stacks.
    -> (strips (n, T + 3, 84, 84) uint8, action (n, T) int32, reward (n, T) float32, h0, h1 (n, hidden) float32,
    notdone (n,) float32, kind: a list of "first" / "mid" / "done" per sequence)."""
    rng = np.random.default_rng(seed)
    cut, drop = int(1.6 * T), T // 2

    def strip(obs, a):
        return obs[np.maximum(0, a - 3 + np.arange(T + 3))]

    def actor():
        while True:
            E = int(rng.integers(episode[0], episode[1] + 1))
            obs = rng.integers(0, 256, (E + 1, 84, 84), dtype=np.uint8)
            start, first = 0, True                    # the buffer holds stacks start .. k - 1
            for k in range(1, E + 1):                 # step k pushes stack k - 1
                if k == E:                            # done: the last stack too, then the buffer's last T
                    yield strip(obs, E + 1 - T), "first" if first else "done", 0.0
                elif k - start == cut:
                    yield strip(obs, start), "first" if first else "mid", 1.0
                    start, first = start + drop, False
                else:
                    yield None

    gens = [actor() for _ in range(actors)]
    out = []
    while len(out) < n:
        for g in gens:
            r = next(g)
            if r is not None and len(out) < n:
                out.append(r)
    strips = np.stack([o[0] for o in out])
    return (strips, rng.integers(0, 6, (n, T)).astype(np.int32), rng.standard_normal((n, T)).astype(np.float32),
            (0.1 * rng.standard_normal((n, hidden))).astype(np.float32),
            (0.1 * rng.standard_normal((n, hidden))).astype(np.float32),
            np.array([o[2] for o in out], np.float32), [o[1] for o in out])
