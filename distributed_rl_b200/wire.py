"""The Redis-facing edge of the three learners: what crosses the actor <-> learner wire and how it
is decoded into the HBM replay's fixed field layouts.

The wire itself (Redis lists / keys of pickled blobs, SURVEY.md §5) is the reference's and is out of
scope; this module only keeps UNMODIFIED actors working against the device-resident learners:

  list  "experience"   Ape-X  [s, a, R_n, s', done, prio]                 APE_X/Player.py:252-261
                       R2D2   [(h0,h1), (s,a,r) x T, done, prio]          R2D2/Player.py:38-63,312-319
  list  "trajectory"   IMPALA [s[T+1,28224], a[T,1], mu[T,1], r[T], flag] IMPALA/Player.py:97-114,183-190
  list  "reward"       episode returns, drained every 500 learner steps   APE_X/Learner.py:219-230
  keys  state_dict / target_state_dict / count / Start                    APE_X/Learner.py:149-155,207-216
        params / Count                                                    IMPALA/Learner.py:286-287

`connect` is anything with redis-py's StrictRedis surface (pipeline / lrange / delete / set / get / scan).
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import torch


def drain(connect, key: str) -> list:
    """Atomically take everything queued under list `key`.

    The reference reads with LRANGE 0 -1 + LTRIM -1 0 inside one MULTI and then DELETEs the key outside
    of it (APE_X/ReplayMemory.py:128-133).  LTRIM -1 0 keeps a ONE-element list intact (start = stop = 0),
    so without the DELETE a lone record is re-read on every poll; with the DELETE outside the transaction,
    records pushed between EXEC and DELETE are lost.  LRANGE + DELETE inside the same MULTI has neither
    problem and is what this does."""
    pipe = connect.pipeline()
    pipe.lrange(key, 0, -1)
    pipe.delete(key)
    return list(pipe.execute()[0] or [])


def wipe_stale_keys(connect, keep=()) -> int:
    """Learner.__init__ (APE_X/Learner.py:41-43, R2D2/Learner.py:54,63-64): drop whatever a previous run
    left in the database (stale `experience`, `Start`, parameters ...).  `keep`: key names that belong to a
    process which is already running beside the learner (a replay server) and are left alone."""
    names = connect.scan()
    keys = list(names[-1]) if names else []
    if keep:
        keep = set(keep)
        keys = [k for k in keys if (k.decode() if isinstance(k, bytes) else k) not in keep]
    if keys:
        connect.delete(*keys)
    return len(keys)


def drain_rewards(connect, default: float = -21.0):
    """Every 500 steps the reference averages and clears the actors' `reward` list
    (APE_X/Learner.py:219-230; -21 when nothing arrived).  -> (mean reward, n)"""
    data = drain(connect, "reward")
    if not data:
        return default, 0
    return float(sum(float(pickle.loads(d)) for d in data) / len(data)), len(data)


def checkpoint_path(log_w: str | None) -> str | None:
    """./weight/<ALG>/<time>/weight.pth (APE_X/Learner.py:256-262); the directory is made on first use."""
    if not log_w:
        return None
    os.makedirs(log_w, exist_ok=True)
    return os.path.join(log_w, "weight.pth")


# ---------------------------------------------------------------------------------------------
# record decoders: pickled actor records -> per-field arrays in the replay's layout
# ---------------------------------------------------------------------------------------------
def decode_apex(recs, out) -> None:
    """recs: unpickled [s, a, R_n, s', done, prio]; out: dict of numpy views s/ns/a/r/d/p (len >= n)."""
    s, ns, a, rw, d, p = (out[k] for k in ("s", "ns", "a", "r", "d", "p"))
    for i, r in enumerate(recs):
        s[i] = np.asarray(r[0], np.uint8).reshape(s.shape[1:])
        ns[i] = np.asarray(r[3], np.uint8).reshape(ns.shape[1:])
        a[i], rw[i], d[i], p[i] = int(r[1]), float(r[2]), bool(r[4]), float(r[5])


def _hidden(h, hidden: int) -> np.ndarray:
    t = h.detach().cpu().numpy() if torch.is_tensor(h) else np.asarray(h)
    return t.reshape(-1)[:hidden].astype(np.float32)


def decode_r2d2(recs, T: int, hidden: int = 512, strip: bool = False):
    """R2D2 records (object arrays): rec[0] = (h0, h1) each (1,1,hidden); rec[1+3t], rec[2+3t], rec[3+3t]
    = s_t (4,84,84) u8, a_t, r_t; rec[-2] = done; rec[-1] = priority.  Exactly the indexing of
    R2D2/ReplayMemory.py:70-88 (`done` becomes notdone = float(not done), :86).
    `strip`: state is written as frame strips (n, T + 3, 84, 84) straight from the records (replay.encode_strip); a
    record whose stacks do not slide raises ValueError naming its position, before anything is returned.
    -> ([state, action, reward, h0, h1, notdone], priorities)"""
    from .replay import encode_strip
    n = len(recs)
    s = np.empty((n, T + 3, 84, 84) if strip else (n, T, 4, 84, 84), np.uint8)
    a = np.empty((n, T), np.int32)
    rw = np.empty((n, T), np.float32)
    h0 = np.empty((n, hidden), np.float32)
    h1 = np.empty((n, hidden), np.float32)
    nd = np.empty(n, np.float32)
    p = np.empty(n, np.float32)
    for i, r in enumerate(recs):
        h0[i], h1[i] = _hidden(r[0][0], hidden), _hidden(r[0][1], hidden)
        if strip:
            encode_strip((r[1 + 3 * t] for t in range(T)), s[i], i)
        for t in range(T):
            if not strip:
                s[i, t] = np.asarray(r[1 + 3 * t], np.uint8).reshape(4, 84, 84)
            a[i, t] = int(r[2 + 3 * t])
            rw[i, t] = float(r[3 + 3 * t])
        nd[i] = float(not r[-2])
        p[i] = float(r[-1])
    return [s, a, rw, h0, h1, nd], p


def decode_impala(recs, T: int):
    """IMPALA rollouts: [s (T+1, 28224) u8, a (T,1), mu (T,1), r (T,), flag] with flag = 0 at episode end
    (IMPALA/Player.py:97-114,176-181; stacked by IMPALA/ReplayMemory.py:34-43).
    -> [state, action, mu, reward, done]  (done keeps the reference's name and meaning: 1 = bootstrap)"""
    n = len(recs)
    s = np.empty((n, T + 1, 4 * 84 * 84), np.uint8)
    a = np.empty((n, T), np.int32)
    mu = np.empty((n, T), np.float32)
    rw = np.empty((n, T), np.float32)
    d = np.empty(n, np.float32)
    for i, r in enumerate(recs):
        s[i] = np.asarray(r[0], np.uint8).reshape(T + 1, -1)
        a[i] = np.asarray(r[1]).reshape(T).astype(np.int32)
        mu[i] = np.asarray(r[2], np.float32).reshape(T)
        rw[i] = np.asarray(r[3], np.float32).reshape(T)
        d[i] = float(r[4])
    return [s, a, mu, rw, d]
