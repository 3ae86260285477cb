"""Numpy restatement of the uniform draw of b2rl_serve_fill_uniform (csrc/serve.cu): B distinct slots of the ring's
valid region [head - size, head), as random.sample draws them (baseline/utils.py:310-315).

Draw k of a fill at Philox counter `offset` is slot (tail + pi(k)) mod capacity, tail = (head - size) mod capacity.
pi is a 4-round balanced Feistel network on the smallest even bit width w >= 2 with 2^w >= size, cycle-walked into
[0, size).  Its round keys are the four words of the Philox4x32-10 block (offset, seed), the generator that
oracle.philox_u01 restates for the sum-tree draws."""
import numpy as np

from oracle.oracle import lowbias32

_M = np.uint64(0xFFFFFFFF)


def philox4x32_10(seed: int, ctr: int) -> np.ndarray:
    """The four uint32 words of one Philox4x32-10 block, counter (ctr_lo, ctr_hi, 0, 0), key = seed."""
    c0, c1 = np.uint64(ctr & 0xFFFFFFFF), np.uint64((ctr >> 32) & 0xFFFFFFFF)
    c2 = c3 = np.uint64(0)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & _M, p1 & _M, ((p0 >> np.uint64(32)) ^ c3 ^ k1) & _M, p0 & _M
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M, (k1 + np.uint64(0xBB67AE85)) & _M
    return np.array([c0, c1, c2, c3], np.uint32)


def feistel_width(size: int) -> int:
    w = 2
    while (1 << w) < size:
        w += 2
    return w


def permutation(seed: int, offset: int, size: int, k) -> np.ndarray:
    """pi(k) for an array of k in [0, size)."""
    key = philox4x32_10(seed, offset)
    half = feistel_width(size) // 2
    mask, sh = np.uint32((1 << half) - 1), np.uint32(half)

    def rounds(x):
        for r in range(4):
            L, R = x >> sh, x & mask
            x = (R << sh) | (L ^ (lowbias32(R ^ key[r]) & mask))
        return x
    y = rounds(np.asarray(k, np.uint32))
    walk = y >= size
    while walk.any():
        y[walk] = rounds(y[walk])
        walk = y >= size
    return y.astype(np.int64)


def uniform_draw(seed: int, offset: int, n: int, size: int, capacity: int, head: int) -> np.ndarray:
    """The n slots b2rl_serve_fill_uniform draws from the device Philox stream at (seed, offset)."""
    if n > size:
        raise ValueError("Sample larger than population")        # what random.sample raises
    tail = (head - size) % capacity
    return (tail + permutation(seed, offset, size, np.arange(n))) % capacity
