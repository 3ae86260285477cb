"""Record the sequences the UNMODIFIED reference R2D2 actor (R2D2/Player.py) sends, as tests/golden/r2d2_actor.npz.

    python tests/golden/make_r2d2_actor_golden.py

Runs in the build container only (the reference is loaded through oracle/ref_harness.py, never copied).  `gym` is
replaced by a stub Atari env whose k-th observation is constant-valued, every pixel k % 251, so frame k of an episode
is recognised by its value after the actor's grey conversion and resize, and the golden stores one byte per frame
instead of 7 056.  Two episodes of 150 and 90 agent steps cover both branches of LocalBuffer.get_traj: the
half-overlap cut at 1.6 * FIXED_TRAJECTORY stacks and the `done` record of each episode's last 80 stacks.

What it stores, per record the actor pushed to `experience`, in push order:
  values   uint8 (n, 80, 4): the value of channel c of stack t (each stack channel is checked to be constant)
  done     bool (n,): the record's `done` flag (rec[-2])
"""
from __future__ import annotations

import os
import pickle
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

EPISODES = (150, 90)        # agent steps per episode (the actor repeats each action over 4 env steps)


class _Stop(Exception):
    pass


class _Env:
    """gym.make('PongNoFrameskip-v4') stand-in: 210 x 160 RGB observations, observation k of the run is constant k % 251;
    no life counter (info lives 0: the actor then ends a life on a non-zero reward, which never comes)."""

    def __init__(self):
        import numpy as np
        self.np, self.k, self.episode, self.t = np, 0, -1, 0

    def seed(self, s):
        pass

    def _obs(self):
        self.k += 1
        return self.np.full((210, 160, 3), self.k % 251, self.np.uint8)

    def reset(self):
        self.episode += 1
        if self.episode == len(EPISODES):
            raise _Stop
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        done = self.t == 4 * EPISODES[self.episode]
        return self._obs(), 0.0, done, {"ale.lives": 0}


class _ObjectArrays:
    """numpy as R2D2/Player.py uses it, except that np.array of a ragged list (LocalBuffer.get_traj's record:
    hidden state, (s, a, r) x T, done) is a 1-D object array, as numpy < 1.24 made it; numpy 2 raises instead."""

    def __init__(self, np):
        self._np = np

    def __getattr__(self, name):
        return getattr(self._np, name)

    def array(self, x, *args, **kwargs):
        try:
            return self._np.array(x, *args, **kwargs)
        except ValueError:
            out = self._np.empty(len(x), object)
            for i, v in enumerate(x):
                out[i] = v
            return out


def main():
    import numpy as np
    import torch
    from oracle import ref_harness as H

    H.enter_reference("r2d2.json")
    gym = types.ModuleType("gym")
    gym.make = lambda name: _Env()
    sys.modules["gym"] = gym
    torch.manual_seed(0)
    np.random.seed(0)
    import R2D2.Player as RP  # type: ignore
    RP.np = _ObjectArrays(np)
    p = RP.Player(idx=0)
    try:
        p.run()
    except _Stop:
        pass
    recs = [pickle.loads(b) for b in p.connect._s.get("experience", [])]
    T = 80
    values, done = [], []
    for r in recs:
        assert len(r) == 1 + 3 * T + 2, len(r)
        st = np.stack([np.asarray(r[1 + 3 * t], np.uint8) for t in range(T)])      # (T, 4, 84, 84)
        v = st[:, :, 0, 0]
        assert (st == v[:, :, None, None]).all(), "a stack channel is not constant"
        values.append(v)
        done.append(bool(r[-2]))
    out = {"values": np.stack(values).astype(np.uint8), "done": np.asarray(done, np.bool_)}
    np.savez_compressed(os.path.join(HERE, "r2d2_actor.npz"), **out)
    print("r2d2_actor.npz:", len(recs), "records, done =", out["done"].tolist())


if __name__ == "__main__":
    main()
