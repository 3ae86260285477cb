"""numpy restatements of the exact-arithmetic tricks the tensor-core kernels rely on (no GPU):
the claims in DESIGN.md §4.6 / §4.9 / §4.10 about what is exact are checked here bit for bit."""
import numpy as np
import pytest


def _wgrad_digits(X):
    """csrc/conv1_wgrad.cu B producers: Y = X + 0x00808080; low three bytes ^ 0x80 are int8 digits, the top byte is q0.
    -> (d0, d1, d2, d3), most significant first."""
    Y = (X + 0x00808080).astype(np.int64)
    assert (Y < 2 ** 31).all() and (Y >= -2 ** 31).all()          # fits the int32 the kernel uses
    Yu = Y.astype(np.int32).view(np.uint32).astype(np.uint32)
    b = [((Yu >> (8 * k)) & 0xFF).astype(np.uint8) for k in range(4)]
    d3, d2, d1 = [(x ^ 0x80).view(np.int8).astype(np.int64) for x in b[:3]]
    return b[3].view(np.int8).astype(np.int64), d1, d2, d3


def _wgrad_digit_scale(absmax):
    """csrc/conv1_wgrad.cu digit_exponent: s = 2^(exponent(fl(max/127)) + 1), the power of two just above max/127."""
    t = np.float32(absmax) / np.float32(127.0)
    e = ((t.view(np.uint32) >> 23) & 0xFF) + 1
    return np.uint32(int(e) << 23).view(np.float32)


def test_balanced_base256_digits_via_bias_reconstruct_exactly():
    """The four digits of _wgrad_digits give back X exactly, the leading one within [-127, 127]."""
    rng = np.random.default_rng(0)
    X = np.concatenate([rng.integers(-(127 << 24), (127 << 24) + 1, size=200000, dtype=np.int64),
                        np.array([0, 1, -1, 127 << 24, -(127 << 24), 128, -128, 0x7F7F7F, -0x808080], np.int64)])
    d0, d1, d2, d3 = _wgrad_digits(X)
    assert (np.abs(d0) <= 127).all()
    assert np.array_equal(((d0 * 256 + d1) * 256 + d2) * 256 + d3, X)


def test_most_negative_wgrad_digits_fit_int32_column_sums():
    """The gradient the GPU test of the accumulators' limit feeds: gy = -0x7E808080 * 2^-24 (fp32-exact; the decimal
    -126.50196087360382 rounds to it) has digit scale 1 and the digits (-126, -128, -128, -128), the most negative
    the bias trick forms.  A CTA's column sum of 160 items of 400 positions of pixel 255 times -128 still fits int32."""
    gy = np.float32(-0x7E808080 * 2.0 ** -24)
    assert float(gy) == -0x7E808080 * 2.0 ** -24 and gy == np.float32(-126.50196087360382)
    s = _wgrad_digit_scale(abs(gy))
    assert s == 1.0
    X = np.array([np.rint(np.float64(gy) / np.float64(s) * 2.0 ** 24)], np.int64)
    assert X[0] == -0x7E808080
    assert [int(d[0]) for d in _wgrad_digits(X)] == [-126, -128, -128, -128]
    assert -128 * 255 * 400 * 160 >= -2 ** 31
    assert -128 * 255 * 400 * 165 < -2 ** 31                      # ... and 165 items would not


def test_power_of_two_scale_keeps_every_gradient_within_127():
    """s = 2^(exponent(fl(max/127)) + 1) > max/127: |v/s| <= 127 and v/s * 2^24 is an exact integer for v >= s."""
    rng = np.random.default_rng(1)
    for _ in range(200):
        v = (rng.standard_normal(400) * 10.0 ** rng.uniform(-6, 3)).astype(np.float32)
        s = _wgrad_digit_scale(np.abs(v).max())
        x = v.astype(np.float64) / np.float64(s) * 2.0 ** 24
        assert np.abs(x).max() <= 127 * 2 ** 24 + 16
        big = np.abs(v) >= s
        assert np.array_equal(x[big], np.rint(x[big]))              # exact integers: no rounding in the digit split
        assert (np.abs(x - np.rint(x)) <= 0.5).all()


def test_tf32_split_is_exact_and_hi_has_ten_mantissa_bits():
    """csrc/gemm.cu split_tf32: hi = rn_tf32(x) by integer add-and-mask, lo = x - hi exactly, hi + lo == x."""
    rng = np.random.default_rng(2)
    x = np.concatenate([(rng.standard_normal(100000) * 10.0 ** rng.uniform(-20, 20, 100000)).astype(np.float32),
                        np.array([0.0, -0.0, 1.0, np.finfo(np.float32).max, np.finfo(np.float32).tiny], np.float32)])
    u = x.view(np.uint32)
    h = ((u.astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32)
    over = (h & 0x7F800000) == 0x7F800000
    h = np.where(over, u & 0xFFFFE000, h)                           # rounding reached inf: truncate instead
    hi = h.view(np.float32)
    lo = (x - hi).astype(np.float32)
    assert (hi.view(np.uint32) & 0x1FFF == 0).all()                 # 10 explicit mantissa bits
    assert np.array_equal((hi.astype(np.float64) + lo.astype(np.float64)).astype(np.float32), x)
    assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), x.astype(np.float64))   # lo is exact
    nz = hi != 0
    assert (np.abs(lo[nz].astype(np.float64)) <= np.abs(hi[nz].astype(np.float64)) * 2.0 ** -10).all()


def test_seven_bit_weight_digits_of_the_forward_kernel():
    """csrc/conv1.cu k_conv1_pack: W = s (q0 + q1/2^7 + q2/2^14 + q3/2^21) to s 2^-22, digits in [-127, 127]."""
    rng = np.random.default_rng(3)
    w = rng.uniform(-0.0625, 0.0625, size=(32, 256)).astype(np.float32)
    w[5, 0] = 0.9
    s = np.abs(w).max(axis=1, keepdims=True).astype(np.float32) / np.float32(127.0)
    x = w.astype(np.float64) / s.astype(np.float64)
    rec = np.zeros_like(x)
    for j in range(4):
        q = np.clip(np.rint(x), -127, 127)
        assert (np.abs(q) <= 127).all()
        rec += q / 128.0 ** j
        x = (x - q) * 128.0
    err = np.abs(rec * s.astype(np.float64) - w.astype(np.float64))
    assert (err <= s.astype(np.float64) * 2.0 ** -22 + 1e-30).all()


def test_int32_accumulator_bound_of_the_wgrad_kernel():
    """MAX_ITEMS_PER_CTA = 160: |sum| <= 128 * 255 * 400 * 160 < 2^31 (digit x pixel x positions x items)."""
    assert 128 * 255 * 400 * 160 < 2 ** 31
    assert 128 * 255 * 400 * 165 >= 2 ** 31


# --------------------------------------------------------------------------- #
# csrc/tree.cu: the sparse (every-4th-level) sum-tree reproduces the binary tree bit for bit    #
# --------------------------------------------------------------------------- #
def _r16_model(p, levels):
    """numpy restatement of csrc/tree.cu's layout: stored level 0 = fp32 leaves, stored level k = binary depth
    levels-4k as fp64, each node = pairwise16 of its (zero-padded) 16 children."""
    cap2 = 1 << levels
    G = (levels + 3) // 4
    top_bits = levels - 4 * (G - 1)
    leaf = np.zeros(cap2, np.float32); leaf[:len(p)] = p
    lv = [leaf.astype(np.float64)]
    for k in range(1, G + 1):
        bits = top_bits if k == G else 4
        c = lv[-1].reshape(-1, 1 << bits)
        c = np.concatenate([c, np.zeros((c.shape[0], 16 - c.shape[1]))], 1)
        s1 = c[:, 0::2] + c[:, 1::2]; s2 = s1[:, 0::2] + s1[:, 1::2]; s3 = s2[:, 0::2] + s2[:, 1::2]
        lv.append(s3[:, 0] + s3[:, 1])
    return lv, G, top_bits


def _r16_descend(lv, G, top_bits, u):
    root = lv[G][0]
    pos = root * u
    node = 0
    for k in range(G, 0, -1):
        bits = top_bits if k == G else 4
        c = np.zeros(16); c[:1 << bits] = lv[k - 1][node << bits:(node + 1) << bits]
        s1 = c[0::2] + c[1::2]; s2 = s1[0::2] + s1[1::2]; s3 = s2[0::2] + s2[1::2]
        ch = 0
        for lvl_sums, width in ((s3, 8), (s2, 4), (s1, 2), (c, 1)):
            base = ch // width          # index of the left child among this level's nodes
            left, right = lvl_sums[base], lvl_sums[base + 1]
            if not (pos < left or right == 0.0):
                pos -= left
                ch += width
        node = (node << bits) | (ch & ((1 << bits) - 1))
    return node


@pytest.mark.parametrize("n", [2, 3, 13, 16, 100, 1000, 4096, 5000, 70000])
def test_sparse_radix16_tree_equals_binary_sumtree(n):
    from oracle import oracle as O
    rng = np.random.default_rng(n)
    p = ((np.abs(rng.standard_normal(n)).clip(max=1) + 1e-7) ** 0.6).astype(np.float32)
    levels = max(1, (n - 1).bit_length())
    lv, G, top_bits = _r16_model(p, levels)
    t = O.SumTreeOracle(1 << levels); t.build(p)
    assert lv[G][0] == t.total                                  # same fp64 root
    for k in range(1, G):                                       # every stored level == the binary tree's level
        d = levels - 4 * k
        np.testing.assert_array_equal(lv[k], t.sum[1 << d:2 << d])
    u = rng.random(300)
    u[:3] = [0.0, 0.5, 1.0 - 2.0 ** -53]
    want, _ = t.sample(u)
    got = np.array([_r16_descend(lv, G, top_bits, x) for x in u])
    np.testing.assert_array_equal(got, want)
