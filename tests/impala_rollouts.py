"""The rollouts the reference IMPALA actors send (IMPALA/Player.py), and the CPU model of the frame-deduplicated IMPALA
store (R.RolloutDedupReplay, DESIGN.md §4.20).

The store pushes a rollout's `state` row as a strip record of R = 4 (T + 1) contiguous frames (csrc/dedup.cu, Strips
layout), so its model is tests/strip_dedup_model.py's StripDedupModel, unchanged, at R = 4 (T + 1): that model takes
R = T' + 3 frames per record, here T' = 4 T + 1."""
from __future__ import annotations

import numpy as np

from dedup_model import ALL_KEY_BITS
from strip_dedup_model import StripDedupModel


def rollout_model(capacity: int, pool_frames: int, window: int, T: int, mask: int = ALL_KEY_BITS) -> StripDedupModel:
    """The CPU model of a RolloutDedupReplay of T-step rollouts: records of R = 4 (T + 1) frames.  Push the rollouts'
    `state` rows as (n, 4 (T + 1), 84, 84) frames (rollout_frames); `strips(slots)` returns them in that shape."""
    return StripDedupModel(capacity, pool_frames, window, 4 * T + 1, mask)


def rollout_frames(state: np.ndarray) -> np.ndarray:
    """(n, T + 1, 28224) rollout rows -> (n, 4 (T + 1), 84, 84): the record's frames in push order."""
    return state.reshape(state.shape[0], -1, 84, 84)


def player_rollouts(n: int, T: int = 20, actors: int = 8, episode=(60, 200), p_done: float = 0.02, seed: int = 0):
    """n rollouts as `actors` reference IMPALA actors send them, interleaved as their episodes progress in lock step.

    An episode of E steps (uniform in `episode`) has observations o_0 .. o_E of random frames; stack k is the last four
    observations o_max(0, k-3) .. o_k (IMPALA/Player.py:88-95, the deque starting as o_0 four times).  A rollout starts
    with a stack s and takes one step per new stack (:151-186); it is sent after T steps, or earlier when a life is
    lost (probability p_done per step, and always at the episode's end) with done = 0, and the next rollout of the
    episode starts with its last stack (:201-203).  checkLength (:116-125) pads a rollout of m < T steps to T + 1
    stacks with stacks m .. T - 1 of the actor's previous rollout (as sent).  An actor's first rollout is never cut
    short, so it always has a previous rollout to pad from.
    -> (state (n, T + 1, 28224) uint8, action (n, T) int32, mu (n, T) float32, reward (n, T) float32, done (n,)
    float32, kind: a list of "first" (an episode's first rollout) / "mid" / "padded" per rollout)."""
    rng = np.random.default_rng(seed)

    def actor():
        past = None
        while True:
            E = int(rng.integers(episode[0], episode[1] + 1))
            obs = rng.integers(0, 256, (E + 1, 84, 84), dtype=np.uint8)
            stacks = obs[np.maximum(0, np.arange(E + 1)[:, None] + np.arange(-3, 1))].reshape(E + 1, 28224)
            cur, first = [0], True                 # stack indices of the rollout being built
            for k in range(1, E + 1):
                cur.append(k)
                m = len(cur) - 1
                cut = k == E or (past is not None and rng.random() < p_done)
                if m < T and not cut:
                    yield None
                    continue
                rows = stacks[cur] if m == T else np.concatenate([past[m:T], stacks[cur]])
                kind = "first" if first else ("mid" if m == T else "padded")
                yield rows, kind, 0.0 if cut else 1.0
                past, first, cur = rows, False, [k]
    gens = [actor() for _ in range(actors)]
    out = []
    while len(out) < n:
        for g in gens:
            r = next(g)
            if r is not None and len(out) < n:
                out.append(r)
    state = np.stack([o[0] for o in out])
    return (state, rng.integers(0, 6, (n, T)).astype(np.int32), rng.uniform(0.05, 0.9, (n, T)).astype(np.float32),
            rng.standard_normal((n, T)).astype(np.float32), np.array([o[2] for o in out], np.float32),
            [o[1] for o in out])
