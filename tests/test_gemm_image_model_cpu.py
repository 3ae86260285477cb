"""The NumPy model of the 3xTF32 operand image and GEMM (tests/gemm_image_model.py), checked on the host: the layout
against the canonical SWIZZLE_64B one, the split at its bit edges, the exactness of exact_operands, and the emulated
GEMM against the exact product, unchanged by the correct reading and changed by every error listed in
gemm_image_model.MUTANTS at the shapes of the exact GPU test (tests/test_gpu_39_gemm_exact.py)."""
import os
import struct

import numpy as np
import pytest

import gemm_image_model as G

SMS = 132       # an H100 SXM; the split count the GPU test realises is asserted there against G.splits


def _packed_floats(rows, k, b_role):
    """b2rl_gemm_packed_floats from the library when it loads on this host, else its statement in the model."""
    try:
        from distributed_rl_b200 import _lib
        return int(_lib.load().b2rl_gemm_packed_floats(rows, k, int(b_role)))
    except Exception:
        return G.packed_floats(rows, k, b_role)


@pytest.mark.parametrize("b_role", [False, True])
@pytest.mark.parametrize("rows,k", [(1, 1), (3, 33), (128, 32), (129, 257), (257, 129), (512, 3136), (1120, 1024)])
def test_offset_is_a_bijection_onto_one_term(rows, k, b_role):
    tr, rp, kc = G.tile_rows(b_role), G.rows_pad(rows, b_role), G.ceil_div(k, G.KC)
    ts = G.term_stride(kc, rp)
    assert 2 * ts == _packed_floats(rows, k, b_role) == G.packed_floats(rows, k, b_role)
    offs = G._unit_offsets(rp, kc, tr)
    assert offs.min() == 0 and offs.max() == ts - 4
    assert (offs % 4 == 0).all()
    assert np.unique(offs).size == offs.size == ts // 4


def _swizzle64(byte_off):
    """CUTLASS Swizzle<2, 4, 3>: address bits [7, 9) XOR-ed into bits [4, 6) (the PTX ISA's 64B swizzle mode)."""
    return byte_off ^ ((byte_off >> 3) & 0x30)


@pytest.mark.parametrize("b_role", [False, True])
def test_each_tile_is_a_canonical_sw64_k_major_operand(b_role):
    """One {term, half-chunk, row tile} tile is tile_rows x 64 B: 8-row x 64-byte atoms 512 B apart (make_desc_sw64's
    stride byte offset), each swizzled as the hardware's 64B mode reads it."""
    tr = G.tile_rows(b_role)
    rp, kc = 3 * tr, 3
    rows = np.arange(rp)[:, None]
    for kh in range(2 * kc):
        for rt in range(rp // tr):
            base = (kh * (rp // tr) + rt) * tr * G.KH
            r = rows[rt * tr:(rt + 1) * tr]
            for unit in range(4):
                got = (G.offset(r, kh * G.KH + 4 * unit, tr, rp) - base) * 4            # bytes inside the tile
                rr = r - rt * tr
                logical = (rr // 8) * 512 + (rr % 8) * 64 + unit * 16                    # row-major 64-byte rows
                assert (got == _swizzle64(logical)).all(), (kh, rt, unit)


def _f(bits):
    return np.array([bits], dtype=np.uint32).view(np.float32)[0]


def _bits(x):
    return int(np.asarray(x, dtype=np.float32).reshape(1).view(np.uint32)[0])


# (input bits, hi bits, lo bits)
_EDGES = [
    (0x00000000, 0x00000000, 0x00000000),          # +0
    (0x80000000, 0x80000000, 0x00000000),          # -0: hi keeps the sign, lo = -0 - -0 = +0
    (0x00000001, 0x00000000, 0x00000001),          # smallest subnormal
    (0x80001FFF, 0x80002000, 0x00000001),          # negative subnormal, rounds up in magnitude
    (0x007FFFFF, 0x00800000, 0x80000001),          # largest subnormal rounds to the smallest normal
    (0x3F801000, 0x3F802000, 0xBA000000),          # 13-bit tie: away from zero, not to even
    (0xBF801000, 0xBF802000, 0x3A000000),          # the same tie, negative
    (0x3F800FFF, 0x3F800000, 0x39FFF000),          # just below the tie
    (0x3F803000, 0x3F804000, 0xBA000000),          # tie with an odd kept bit
    (0x7F7FEFFF, 0x7F7FE000, 0x797FF000),          # the largest float whose hi is finite after rounding
    (0x7F7FF000, 0x7F7FE000, 0x79800000),          # rounding reaches inf: truncated
    (0x7F7FFFFF, 0x7F7FE000, 0x79FFF800),          # FLT_MAX: truncated
    (0xFF7FFFFF, 0xFF7FE000, 0xF9FFF800),          # -FLT_MAX
    (0x7F800000, 0x7F800000, 0x00000000),          # +inf
    (0xFF800000, 0xFF800000, 0x00000000),          # -inf
    (0x7FC00000, 0x7FC00000, 0x00000000),          # quiet NaN
    (0x7FC01234, 0x7FC01234, 0x00000000),          # quiet NaN with a payload in the dropped bits
    (0xFFFFFFFF, 0xFFFFFFFF, 0x00000000),          # negative NaN, all payload bits: u + 0x1000 wraps
    (0x7F800001, 0x7F800001, 0x00000000),          # signalling NaN
    (0xFFA00FFF, 0xFFA00FFF, 0x00000000),          # signalling NaN, negative, payload
]


def test_the_special_values_are_the_split_edges():
    assert list(G.SPECIAL_BITS) == [e[0] for e in _EDGES]


@pytest.mark.parametrize("x,hi,lo", _EDGES, ids=[f"{e[0]:08x}" for e in _EDGES])
def test_split_tf32_edges(x, hi, lo):
    h, l_ = G.split_tf32(np.array([x], dtype=np.uint32).view(np.float32))
    assert (_bits(h), _bits(l_)) == (hi, lo), (hex(_bits(h)), hex(_bits(l_)))
    assert _bits(h) & 0x1FFF == 0 or not np.isfinite(_f(x))
    if np.isfinite(_f(x)):
        assert float(h[0]) + float(l_[0]) == float(_f(x))


def test_split_tf32_is_exact_on_random_bits():
    bits = np.random.default_rng(0).integers(0, 2 ** 32, size=1 << 18, dtype=np.uint64).astype(np.uint32)
    x = bits.view(np.float32)
    h, l_ = G.split_tf32(x)
    fin = np.isfinite(x)
    assert ((h[fin].view(np.uint32) & 0x1FFF) == 0).all()
    assert (h[fin].astype(np.float64) + l_[fin].astype(np.float64) == x[fin].astype(np.float64)).all()
    # hi is the nearest TF32 value (ties away from zero) unless that rounds to inf: |lo| <= half its ulp
    ulp = np.spacing(np.abs(h[fin]).astype(np.float32)).astype(np.float64) * 2 ** 13
    ok = np.isfinite(ulp) & (np.abs(h[fin]) < np.float32(3.4e38))
    assert (np.abs(l_[fin][ok].astype(np.float64)) <= ulp[ok] / 2).all()
    assert (h[~fin].view(np.uint32) == bits[~fin]).all() and (l_[~fin] == 0).all()


@pytest.mark.parametrize("M,N,K", [(63, 5, 3136), (129, 257, 129), (1, 3, 3136), (257, 1, 33)])
def test_exact_operands_sum_exactly_in_any_order(M, N, K):
    """Every output of exact_operands' 3xTF32 product, summed in fp32 in 50 random orders and by random split
    partitions (each part summed, then the parts in order), is the fp64 sum bit for bit."""
    a, b = G.exact_operands(M, N, K, seed=M + N + K)
    exact = G.exact_product(a, b)
    assert (exact.astype(np.float32).astype(np.float64) == exact).all()
    a_hi, a_lo = G.split_tf32(a)
    b_hi, b_lo = G.split_tf32(b)
    rng = np.random.default_rng(1)
    for _ in range(3):
        m, n = rng.integers(M), rng.integers(N)
        terms = np.concatenate([a_lo[m] * b_hi[n], a_hi[m] * b_lo[n], a_hi[m] * b_hi[n]]).astype(np.float32)
        assert (terms.astype(np.float64) == np.concatenate(
            [a_lo[m].astype(np.float64) * b_hi[n], a_hi[m].astype(np.float64) * b_lo[n],
             a_hi[m].astype(np.float64) * b_hi[n]])).all()                # each product exact in fp32
        for _ in range(50):
            t = terms[rng.permutation(terms.size)]
            s = np.float32(0.0)
            for v in t:
                s = np.float32(s + v)
            assert float(s) == exact[m, n]
            cuts = np.sort(rng.choice(np.arange(1, t.size), size=min(7, t.size - 1), replace=False))
            parts = [np.float32(0.0)]
            for piece in np.split(t, cuts):
                p = np.float32(0.0)
                for v in piece:
                    p = np.float32(p + v)
                parts.append(p)
            total = np.float32(0.0)
            for p in parts:
                total = np.float32(total + p)
            assert float(total) == exact[m, n]


def test_exact_operands_cover_every_half_chunk_and_swizzle_unit():
    for M, K in [(128, 3136), (63, 3136), (257, 129), (1, 3136), (2, 20480 // 8)]:
        mask = G.sparse_pattern(M, K)
        for cov in G.coverage(mask, K):
            reach = min(len(cov["all_halves"]), cov["rows"] * G.MAX_NNZ)
            assert len(cov["halves"]) == reach
            if cov["rows"] >= 8:
                assert cov["pairs"] == cov["all_pairs"]
        assert mask.sum(1).max() <= G.MAX_NNZ


def test_splits_follow_gemm_splits():
    """The split counts recorded with tests/golden/gemm_tf32x3_sm90.json on 132 SMs."""
    import json
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_tf32x3_sm90.json")) as f:
        rec = json.load(f)
    for e in rec["shapes"]:
        if "splits" in e:
            assert G.splits(e["M"], e["N"], e["K"], rec["sms"]) == e["splits"], e["name"]
    assert G.splits(256, 2592, 20480, 132) == 20           # 640 chunks: the 32-chunk cap sets it
    assert G.splits(1, 1, 33 * 32, 132) == 33 and G.depths(33 * 32, 33) == [2] * 33
    assert G.splits(1, 1, 3136, 132) == 98                  # 98 chunks, 132 SMs: one chunk per split
    assert G.depths(100 * 32, G.splits(1, 1, 100 * 32, 7)) == [30] * 6 + [20]    # 7 splits of 15 chunks, the last 10
    for nk, K in G.DEPTH_K.items():
        for sms in (114, 132, 144):
            assert G.splits(G.DEPTH_M, G.DEPTH_N, K, sms) == 1
            assert G.depths(K, 1) == [nk]


def _emulation_grid():
    grid = [(G.DEPTH_M, G.DEPTH_N, K, None) for K in G.DEPTH_K.values()]
    return grid + G.edge_shapes()


def _ids(g):
    return [f"{M}x{N}x{K}" for M, N, K, _ in g]


@pytest.mark.parametrize("M,N,K,ldc", _emulation_grid(), ids=_ids(_emulation_grid()))
def test_emulated_gemm_is_exact_and_every_mutant_changes_it(M, N, K, ldc):
    a, b = G.exact_operands(M, N, K, seed=M * 7 + N * 13 + K)
    exact = G.exact_product(a, b)
    a_img, b_img = G.image(a, False, False), G.image(b, False, True)
    n_splits = G.splits(M, N, K, SMS)
    parts, total = G.emulate(a_img, b_img, M, N, K, SMS)
    assert parts.shape[0] == n_splits
    assert (total == exact).all()
    for z in range(n_splits):
        c0, c1 = G.split_range(K, n_splits, z)
        k0, k1 = c0 * G.KC, min(c1 * G.KC, K)
        assert (parts[z] == G.exact_product(a[:, k0:k1], b[:, k0:k1])).all()
    wraps = max(G.depths(K, n_splits)) > G.STAGES
    for mutant in G.MUTANTS:
        mp, mt = G.emulate(a_img, b_img, M, N, K, SMS, mutant)
        changed = (mp != parts).any() or (mt != total).any()
        if mutant == "stale_stage" and not wraps:
            assert not changed          # the ring never wraps at this depth: nothing stale to read
            continue
        if mutant == "no_xor" and max(M, N) <= 2:
            assert not changed          # rows 0 and 1 are not swizzled
            continue
        assert changed, mutant


def test_stale_stage_mutant_is_reachable():
    """The stale-stage mutant needs a split deeper than the ring; the depth grid has them."""
    deep = [nk for nk, K in G.DEPTH_K.items() if max(G.depths(K, 1)) > G.STAGES]
    assert deep == [6, 8, 10, 16, 64]


def test_special_values_pack_through_the_model():
    """The edge values of the split, in one image row: hi and lo land in their units, NaN payloads unchanged."""
    vals = np.array(G.SPECIAL_BITS, dtype=np.uint32).view(np.float32)
    img = G.image(vals[None, :], False, False)
    hi, lo = G.read_image(img, 1, vals.size, False)
    h, l_ = G.split_tf32(vals)
    assert (hi[0, :vals.size].view(np.uint32) == h.view(np.uint32)).all()
    assert (lo[0, :vals.size].view(np.uint32) == l_.view(np.uint32)).all()
    assert (hi[1:] == 0).all() and (hi[0, vals.size:] == 0).all()
    assert struct.pack("<f", 0.0) == hi[0, vals.size:vals.size + 1].tobytes()
