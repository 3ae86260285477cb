"""numpy restatement of the frame codec of the compressed R2D2 frame pool (csrc/frame_codec.cuh, DESIGN.md §4.21), a
deterministic Atari-like frame source, and a CPU model of the coded store's unit ring.

encode / decode state the byte format the kernels write and read.  atari_frame renders a synthetic frame: flat
background, walls, a brick band, two paddles, a ball and score digits, all moving with the step.  atari_sequences
cuts those frames into sequences with the actor structure of strip_dedup_model.player_sequences.  CodedStripDedupModel
is StripDedupModel with the frames stored encoded in a ring of P 16-byte units and the byte twin of the eviction rule.
Every number here is for synthetic frames, not for frames of a real Atari emulator."""
from __future__ import annotations

import numpy as np

from strip_dedup_model import MAX_FRAMES, StripDedupModel

SIDE, FRAME = 84, 84 * 84
HEADER, MASK = 16, 11
RAW_UNITS = (HEADER + FRAME) // 16          # 442
RAW_BYTES = 16 * RAW_UNITS                  # 7 072
RAW, ROWRUN = 0, 1


def _header(kind: int, units: int, repeat_mask: np.ndarray) -> np.ndarray:
    h = np.zeros(HEADER, np.uint8)
    h[0], h[1], h[2] = kind, units & 0xFF, units >> 8
    h[3:14] = repeat_mask
    return h


def encode(frame) -> np.ndarray:
    """The encoding of one 84 x 84 uint8 frame: a multiple of 16 bytes, at most 7 072."""
    f = np.asarray(frame, np.uint8).reshape(SIDE, SIDE)
    rep = np.zeros(SIDE, bool)
    rep[1:] = (f[1:] == f[:-1]).all(1)
    change = np.ones((SIDE, SIDE), bool)
    change[:, 1:] = f[:, 1:] != f[:, :-1]
    coded = np.flatnonzero(~rep)
    masks = np.packbits(change[coded], axis=1, bitorder="little")        # (C, 11), bits 84..87 zero
    lits = f[coded][change[coded]]
    nbytes = HEADER + MASK * len(coded) + len(lits)
    units = -(-nbytes // 16)
    if units >= RAW_UNITS:
        return np.concatenate([_header(RAW, RAW_UNITS, np.zeros(MASK, np.uint8)), f.ravel()])
    body = np.concatenate([_header(ROWRUN, units, np.packbits(rep, bitorder="little")), masks.ravel(), lits])
    return np.concatenate([body, np.zeros(16 * units - nbytes, np.uint8)])


def units(frame) -> int:
    return len(encode(frame)) // 16


def decode(enc) -> np.ndarray:
    e = np.asarray(enc, np.uint8)
    if e[0] == RAW:
        return e[HEADER:HEADER + FRAME].reshape(SIDE, SIDE).copy()
    assert e[0] == ROWRUN
    rep = np.unpackbits(e[3:14], bitorder="little")[:SIDE].astype(bool)
    C = SIDE - int(rep.sum())
    masks = np.unpackbits(e[HEADER:HEADER + MASK * C].reshape(C, MASK), axis=1, bitorder="little")[:, :SIDE].astype(np.int64)
    counts = masks.sum(1).astype(np.int64)
    base = HEADER + MASK * C + np.concatenate([[0], np.cumsum(counts)[:-1]])
    k = np.arange(SIDE) - np.cumsum(rep)                                   # the coded row each row repeats
    idx = base[k][:, None] + np.cumsum(masks[k], axis=1) - 1
    return e[idx]


# ---- a synthetic Atari-like frame source ---------------------------------------------------------------------------
_DIGITS = ["111101101101111", "010110010010111", "111001111100111", "111001111001111", "101101111001001",
           "111100111001111", "111100111101111", "111001001001001", "111101111101111", "111101111001111"]


def _bounce(p: int, lo: int, hi: int) -> int:
    """p folded into [lo, hi] as a ball bouncing between two walls."""
    span = hi - lo
    q = p % (2 * span)
    return lo + (q if q <= span else 2 * span - q)


def atari_frame(k: int, episode: int = 0) -> np.ndarray:
    """Frame k of synthetic episode `episode`, a deterministic function of both, in the style of a preprocessed
    (84 x 84 grayscale) Atari frame: flat background, a top bar and side walls, a band of six rows of bricks (one
    disappearing every few steps), two paddles, a 2 x 2 ball and a three-digit score."""
    rng = np.random.default_rng(episode)
    x0, y0, vx, vy, p0, q0 = (int(v) for v in rng.integers(0, 1000, 6))
    f = np.zeros((SIDE, SIDE), np.uint8)
    f[:, :4] = f[:, 80:] = 142                                             # side walls
    f[8:11, :] = 142                                                       # the top bar
    shades = (200, 180, 160, 140, 120, 100)
    gone = rng.permutation(6 * 19)[:min(6 * 19, k // 7)]                   # bricks hit so far
    alive = np.ones(6 * 19, bool)
    alive[gone] = False
    for i in range(6):
        for j in range(19):
            if alive[i * 19 + j]:
                f[20 + 2 * i:22 + 2 * i, 4 + 4 * j:8 + 4 * j] = shades[i]
    bx = _bounce(x0 + (1 + vx % 3) * k, 4, 78)
    by = _bounce(y0 + (1 + vy % 2) * k, 34, 74)
    f[by:by + 2, bx:bx + 2] = 236                                          # the ball
    px = _bounce(p0 + 2 * k, 4, 68)
    f[76:78, px:px + 12] = 200                                             # the bottom paddle
    qy = _bounce(q0 + k, 34, 66)
    f[qy:qy + 8, 5:7] = 90                                                 # a side paddle
    score = (k // 5) % 1000
    for d, c in enumerate(f"{score:03d}"):                                 # the score, 3 x 5 digits at 2x
        g = np.array([int(b) for b in _DIGITS[int(c)]], np.uint8).reshape(5, 3) * 230
        f[1:11:2, 30 + 8 * d:36 + 8 * d:2][:g.shape[0], :g.shape[1]] = np.maximum(
            f[1:11:2, 30 + 8 * d:36 + 8 * d:2][:g.shape[0], :g.shape[1]], g)
        f[2:11:2, 30 + 8 * d:36 + 8 * d:2][:5, :3] = f[1:11:2, 30 + 8 * d:36 + 8 * d:2][:5, :3]
        f[1:11, 31 + 8 * d:37 + 8 * d:2] = f[1:11, 30 + 8 * d:36 + 8 * d:2]
    return f


def atari_sequences(n: int, T: int = 80, actors: int = 4, episode=(120, 400), seed: int = 0, hidden: int = 512):
    """player_sequences (strip_dedup_model) with atari_frame observations in place of random ones: the same actor
    structure (stacks of the last four observations, sequences cut at int(1.6 T) stacks with T / 2 dropped, the
    episode's last T stacks at its end), episodes interleaved across `actors`.  Returns what player_sequences does."""
    rng = np.random.default_rng(seed)
    cut, drop = int(1.6 * T), T // 2
    episodes = iter(range(seed * 1_000_003, seed * 1_000_003 + 1_000_000))

    def strip(obs, a):
        return obs[np.maximum(0, a - 3 + np.arange(T + 3))]

    def actor():
        while True:
            E = int(rng.integers(episode[0], episode[1] + 1))
            ep = next(episodes)
            obs = np.stack([atari_frame(k, ep) for k in range(E + 1)])
            start, first = 0, True
            for k in range(1, E + 1):
                if k == E:
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


# ---- the coded store -----------------------------------------------------------------------------------------------
def coded_max_batch(capacity: int, pool_frames: int, window: int, R: int, pool_units: int) -> int:
    """Sequences per push of a coded store (b2rl_dedup_info): the frame bound, and the unit bound
    (P - (W + 2) 442) / (442 R)."""
    return min(capacity, (pool_frames - window - 1) // R, MAX_FRAMES // R,
               (pool_units - (window + 2) * RAW_UNITS) // (R * RAW_UNITS))


class CodedStripDedupModel(StripDedupModel):
    """StripDedupModel with the frames stored encoded in a ring of `pool_units` 16-byte units: frame seq's entry
    seq % F is (absolute unit offset, units); a frame that would straddle the ring's end starts at the next multiple of
    P and the skipped units count as written; a slot also dies once P - (W + 1) 442 units have been written since its
    batch began.  Hits compare the decoded stored frame, and strips() decodes from the ring."""

    def __init__(self, capacity: int, pool_frames: int, window: int, T: int, pool_units: int, **kw):
        super().__init__(capacity, pool_frames, window, T, **kw)
        self.P = pool_units
        self.ring = np.zeros(16 * pool_units, np.uint8)
        self.units = 0                         # units written so far
        self.foff = np.zeros(pool_frames, np.int64)
        self.flen = np.zeros(pool_frames, np.int64)
        self.uins = np.zeros(capacity, np.int64)

    def stored(self, entry: int) -> np.ndarray:
        a = 16 * (int(self.foff[entry]) % self.P)
        return decode(self.ring[a:a + 16 * int(self.flen[entry])])

    def push(self, strips: np.ndarray, prio: np.ndarray) -> None:
        mb = coded_max_batch(self.cap, self.F, self.W, self.R, self.P)
        for a in range(0, len(prio), mb):
            self._push(strips[a:a + mb], prio[a:a + mb])

    def _push(self, strips, prio):
        from dedup_model import frame_keys
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
            if c >= 0 and c >= head - self.W and np.array_equal(self.stored(c % self.F), frames[j]):
                seq[j] = c
        misses = [j for j in range(R * n) if rep[j] == j and seq[j] < 0]
        encs, offs, U = [], [], self.units
        for r, j in enumerate(misses):
            seq[j] = head + r
            e = encode(frames[j])
            u = len(e) // 16
            if U % self.P + u > self.P:            # never straddle the ring's end
                U += self.P - U % self.P
            encs.append(e)
            offs.append(U)
            U += u
        head_new, units_new = head + len(misses), U
        tail = (self.slot_head - self.size) % self.cap
        while self.size > 0 and (head_new - self.ins[tail] >= self.F - self.W
                                 or units_new - self.uins[tail] >= self.P - (self.W + 1) * RAW_UNITS):
            self.prio[tail] = 0.0
            tail = (tail + 1) % self.cap
            self.size -= 1
        for j, e, off in zip(misses, encs, offs):
            ent = seq[j] % self.F
            a = 16 * (off % self.P)
            self.ring[a:a + len(e)] = e
            self.foff[ent], self.flen[ent] = off, len(e) // 16
            self.pool[ent] = frames[j]
            self.table[int(keys[j])] = max(self.table.get(int(keys[j]), -1), int(seq[j]))
        for i in range(n):
            slot = (self.slot_head + i) % self.cap
            self.planes[slot] = seq[rep[R * i:R * i + R]] % self.F
            self.ins[slot] = head
            self.uins[slot] = self.units
            self.prio[slot] = prio[i]
        self.slot_head = (self.slot_head + n) % self.cap
        self.size = min(self.size + n, self.cap)
        self.head, self.units = head_new, units_new
        self.new_frames.append(len(misses))

    def strips(self, slots) -> np.ndarray:
        """The (m, T + 3, 84, 84) strips of `slots`, decoded from the unit ring."""
        p = self.planes[np.asarray(slots)]
        return np.stack([np.stack([self.stored(int(e)) for e in row]) for row in p.reshape(-1, self.R)]).reshape(
            p.shape + (84, 84))
