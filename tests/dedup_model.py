"""CPU model of the frame-deduplicated Ape-X store (DESIGN.md §4.16, csrc/dedup.cu) and a generator of the records
the reference actor sends (APE_X/Player.py).

The model keeps the rule, not the kernels: the 64-bit frame key, the lowest-position rule inside a batch, the window,
the sequence numbers of the misses in batch order, and both eviction conditions.  The GPU store must give the same
pool ids, liveness and priorities for the same record stream."""
from __future__ import annotations

import numpy as np

FRAME = 84 * 84
ALL_KEY_BITS = (1 << 63) - 1
_M1, _M2, _GOLD = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB), np.uint64(0x9E3779B97F4A7C15)


def _mix64(z: np.ndarray) -> np.ndarray:
    z = z ^ (z >> np.uint64(30))
    z = z * _M1
    z = z ^ (z >> np.uint64(27))
    z = z * _M2
    return z ^ (z >> np.uint64(31))


def frame_keys(frames: np.ndarray, mask: int = ALL_KEY_BITS) -> np.ndarray:
    """(m, 84, 84) uint8 -> uint64[m]: mix64(sum_i mix64(w_i ^ i * golden)) & mask, top bit cleared, w_i the
    frame's little-endian 8-byte words (the key k_dedup_hash computes)."""
    w = np.ascontiguousarray(frames, np.uint8).reshape(len(frames), FRAME).view("<u8")
    with np.errstate(over="ignore"):
        h = _mix64(w ^ (np.arange(w.shape[1], dtype=np.uint64) * _GOLD)).sum(axis=1, dtype=np.uint64)
        return _mix64(h) & np.uint64(mask & ALL_KEY_BITS)


def max_batch(capacity: int, pool_frames: int, window: int) -> int:
    """Records per push (b2rl_dedup_info): larger pushes are split into chunks of this many."""
    return min(capacity, (pool_frames - window - 1) // 8, 8192)


class DedupModel:
    def __init__(self, capacity: int, pool_frames: int, window: int, mask: int = ALL_KEY_BITS):
        self.cap, self.F, self.W, self.mask = capacity, pool_frames, window, mask
        self.pool = np.zeros((pool_frames, 84, 84), np.uint8)
        self.table = {}                       # key -> seq of the newest frame stored under it
        self.head = 0                         # frames stored so far
        self.slot_head, self.size = 0, 0
        self.ins = np.zeros(capacity, np.int64)
        self.planes = np.zeros((capacity, 8), np.int32)
        self.prio = np.zeros(capacity, np.float32)
        self.new_frames = []                  # frames stored per pushed chunk

    def push(self, s: np.ndarray, ns: np.ndarray, prio: np.ndarray) -> None:
        mb = max_batch(self.cap, self.F, self.W)
        for a in range(0, len(prio), mb):
            self._push(s[a:a + mb], ns[a:a + mb], prio[a:a + mb])

    def _push(self, s, ns, prio):
        n = len(prio)
        frames = np.concatenate([np.asarray(s, np.uint8).reshape(n, 4, 84, 84),
                                 np.asarray(ns, np.uint8).reshape(n, 4, 84, 84)], axis=1).reshape(8 * n, 84, 84)
        keys = frame_keys(frames, self.mask)
        first, seq = {}, np.full(8 * n, -1, np.int64)
        rep = np.arange(8 * n)
        head = self.head
        for j, k in enumerate(keys.tolist()):
            f = first.setdefault(k, j)
            if f < j and np.array_equal(frames[f], frames[j]):
                rep[j] = f
                continue
            c = self.table.get(k, -1)
            if c >= 0 and c >= head - self.W and np.array_equal(self.pool[c % self.F], frames[j]):
                seq[j] = c
        misses = [j for j in range(8 * n) if rep[j] == j and seq[j] < 0]
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
            self.planes[slot] = seq[rep[8 * i:8 * i + 8]] % self.F
            self.ins[slot] = head
            self.prio[slot] = prio[i]
        self.slot_head = (self.slot_head + n) % self.cap
        self.size = min(self.size + n, self.cap)
        self.head = head_new
        self.new_frames.append(len(misses))

    def live_slots(self) -> np.ndarray:
        return (self.slot_head - self.size + np.arange(self.size)) % self.cap

    def stacks(self, slots) -> tuple:
        """The (s, s') stacks the pool ids of `slots` name."""
        p = self.pool[self.planes[np.asarray(slots)]]            # (m, 8, 84, 84)
        return p[:, :4], p[:, 4:]


def player_records(n: int, actors: int = 8, episode: int = 40, unroll: int = 3, seed: int = 0, chunk: int = 5):
    """n records as `actors` reference actors send them, interleaved `chunk` records at a time: episodes of
    `episode` random frames; each step's stack is the last four frames, an episode starting with its first frame four
    times (APE_X/Player.py:203-209); LocalBuffer.get_traj (:33-57) pairs stack t with stack t + unroll (with the
    episode's last stack near its end, done = 1).  -> s, ns (n, 4, 84, 84) uint8, a int32, r float32, d uint8."""
    rng = np.random.default_rng(seed)

    def actor():
        while True:
            frames = rng.integers(0, 256, (episode, 84, 84), dtype=np.uint8)
            stacks = [np.stack([frames[max(0, t - 3 + i)] for i in range(4)]) for t in range(episode)]
            for t in range(episode):
                u = min(t + unroll, episode - 1)
                yield stacks[t], stacks[u], int(rng.integers(6)), float(rng.standard_normal()), int(u == episode - 1)

    gens = [actor() for _ in range(actors)]
    out = []
    k = 0
    while len(out) < n:
        for _ in range(chunk):
            out.append(next(gens[k]))
        k = (k + 1) % actors
    out = out[:n]
    s = np.stack([o[0] for o in out])
    ns = np.stack([o[1] for o in out])
    return (s, ns, np.array([o[2] for o in out], np.int32), np.array([o[3] for o in out], np.float32),
            np.array([o[4] for o in out], np.uint8))
