"""Player-like Ape-X records built from the synthetic Atari-like frames of pool_codec_model.atari_frame: stacks of the
last four frames (an episode starts with its first frame four times, APE_X/Player.py:203-209), s' the stack
UNROLL_STEP steps later (LocalBuffer.get_traj, :33-57), actors interleaved a few records at a time."""
import numpy as np

from pool_codec_model import atari_frame


def atari_records(n: int, actors: int = 8, episode: int = 40, unroll: int = 3, seed: int = 0, chunk: int = 5):
    """-> s, ns (n, 4, 84, 84) uint8, a int32, r float32, d uint8, as dedup_model.player_records."""
    rng = np.random.default_rng(seed)
    episodes = iter(range(seed * 1000, 10 ** 9))

    def actor():
        while True:
            e = next(episodes)
            frames = [atari_frame(k, e) for k in range(episode)]
            stacks = [np.stack([frames[max(0, t - 3 + i)] for i in range(4)]) for t in range(episode)]
            for t in range(episode):
                u = min(t + unroll, episode - 1)
                yield stacks[t], stacks[u], int(rng.integers(6)), float(rng.standard_normal()), int(u == episode - 1)

    gens = [actor() for _ in range(actors)]
    out, k = [], 0
    while len(out) < n:
        for _ in range(chunk):
            out.append(next(gens[k]))
        k = (k + 1) % actors
    out = out[:n]
    return (np.stack([o[0] for o in out]), np.stack([o[1] for o in out]), np.array([o[2] for o in out], np.int32),
            np.array([o[3] for o in out], np.float32), np.array([o[4] for o in out], np.uint8))
