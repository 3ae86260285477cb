"""Player-like IMPALA rollouts built from the synthetic Atari-like frames of pool_codec_model.atari_frame, for the coded
rollout store (R.RolloutDedupReplay(pool_bytes=...), DESIGN.md §4.23): the actor structure of
impala_rollouts.player_rollouts (stacks of the last four observations, rollouts of T steps sharing their boundary stack,
short rollouts padded by checkLength with the previous rollout's stacks, actors interleaved) with compressible
observations in place of random ones."""
from __future__ import annotations

import numpy as np

from pool_codec_model import atari_frame


def atari_rollouts(n: int, T: int = 20, actors: int = 8, episode=(60, 200), p_done: float = 0.02, seed: int = 0):
    """-> what impala_rollouts.player_rollouts returns: state (n, T + 1, 28224) uint8, action (n, T) int32, mu and
    reward (n, T) float32, done (n,) float32, and the kind of each rollout."""
    rng = np.random.default_rng(seed)
    episodes = iter(range(seed * 1_000_003, seed * 1_000_003 + 1_000_000))

    def actor():
        past = None
        while True:
            E = int(rng.integers(episode[0], episode[1] + 1))
            ep = next(episodes)
            obs = np.stack([atari_frame(k, ep) for k in range(E + 1)])
            stacks = obs[np.maximum(0, np.arange(E + 1)[:, None] + np.arange(-3, 1))].reshape(E + 1, 28224)
            cur, first = [0], True
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


def staging_map(planes: np.ndarray, F: int) -> np.ndarray:
    """The staged plane table of b2rl_dedup_stage_rollouts for drawn rows `planes` (n, R) of pool ids: entry (k, c) is
    k R + i, i the first position of row k whose id (mod F, as an unsigned 32-bit value) equals position c's."""
    ids = np.asarray(planes, np.int32).astype(np.uint32).astype(np.int64) % F
    n, R = ids.shape
    out = np.empty((n, R), np.int32)
    for k in range(n):
        first = {}
        for c in range(R):
            out[k, c] = k * R + first.setdefault(int(ids[k, c]), c)
    return out
