"""Every 3xTF32 operand-image writer and the GEMM (csrc/gemm.cu, csrc/optim.cu) bit for bit against the NumPy model in
tests/gemm_image_model.py.

Writers: every output buffer starts as a NaN pattern, so a unit that a writer leaves unwritten, padding included, fails
the comparison.  GEMM: the operands come from gemm_image_model.exact_operands, whose 3xTF32 product is exact in fp32 at
every intermediate, so the correct result is one bit pattern whatever the split count, the accumulation order or the
SM count.  A missing, doubled or misplaced term changes bits; tests/test_gemm_image_model_cpu.py shows that for each
layout, pipeline and split error in gemm_image_model.MUTANTS.  The split count is asserted against the model for this
card's SM count, so nothing here skips on another count."""
import numpy as np
import pytest

import gemm_image_model as G

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

NAN_BITS = 0x7FBADBAD          # a signalling-NaN payload no writer produces
SENTINEL_BITS = 0x7FC0FFEE     # fills the GEMM's guard rows and columns


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def lib(dev):
    from distributed_rl_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _filled(n, bits=NAN_BITS):
    return torch.full((n,), bits, dtype=torch.int32, device="cuda").view(torch.float32)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _assert_bits(got: torch.Tensor, want: np.ndarray, what):
    want_t = torch.from_numpy(np.ascontiguousarray(want, dtype=np.float32).view(np.int32)).to(got.device)
    got_i = got.contiguous().view(torch.int32)
    assert got_i.shape == want_t.shape, (what, tuple(got_i.shape), tuple(want_t.shape))
    bad = (got_i != want_t).nonzero()
    if bad.numel():
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} floats differ, first at {i}: "
                             f"got {int(got_i[i]) & 0xFFFFFFFF:08x}, want {int(want_t[i]) & 0xFFFFFFFF:08x}")


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()


# --------------------------------------------------------------------------------------------------------------------- #
# writers                                                                                                               #
# --------------------------------------------------------------------------------------------------------------------- #
def _writer_pairs():
    """(src_rows, src_cols): every size of WRITER_SIZES as rows with three contraction lengths."""
    s = G.WRITER_SIZES
    return [(s[i], s[(i + d) % len(s)]) for i in range(len(s)) for d in (0, 5, 9)]


def _split_pack(lib, src_flat, src_off, rows, cols, ld, transpose, b_role):
    """b2rl_gemm_split_pack of the rows x cols matrix at element src_off of src_flat (leading dimension ld) into a
    NaN-filled image."""
    op_rows, op_k = (cols, rows) if transpose else (rows, cols)
    out = _filled(G.packed_floats(op_rows, op_k, b_role))
    lib.check(lib.load().b2rl_gemm_split_pack(src_flat.data_ptr() + 4 * src_off, rows, cols, ld, int(transpose),
                                              int(b_role), out.data_ptr(), _stream()))
    return out


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("b_role", [False, True])
def test_split_pack_matches_the_model(lib, transpose, b_role):
    """Every size of the writers' list as rows and as contraction, in three source layouts: contiguous, a leading
    dimension wider than the row, and a source pointer 4 bytes past a 16-byte boundary (the unaligned path)."""
    rng = np.random.default_rng(int(transpose) * 2 + int(b_role))
    for q, (rows, cols) in enumerate(_writer_pairs()):
        layout = q % 3
        ld = cols + 3 if layout == 1 else cols
        off = 1 if layout == 2 else 0
        mat = rng.standard_normal((rows, cols)).astype(np.float32)
        flat = np.full(off + rows * ld + 4, np.nan, dtype=np.float32)
        flat[off:off + rows * ld].reshape(rows, ld)[:, :cols] = mat
        got = _split_pack(lib, _cuda(flat), off, rows, cols, ld, transpose, b_role)
        _assert_bits(got, G.image(mat, transpose, b_role), (rows, cols, ld, off))


def _special_matrix(rows, cols, seed):
    """Standard normal, with every value of G.SPECIAL_BITS at four random places."""
    rng = np.random.default_rng(seed)
    m = rng.standard_normal((rows, cols)).astype(np.float32)
    flat = m.reshape(-1).view(np.uint32)
    pos = rng.choice(flat.size, size=4 * len(G.SPECIAL_BITS), replace=False)
    flat[pos] = np.tile(np.array(G.SPECIAL_BITS, dtype=np.uint32), 4)
    return m


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("b_role", [False, True])
def test_split_pack_special_values(lib, transpose, b_role):
    """Signed zeros, subnormals, the 13-bit ties, the largest finite values, infinities and NaNs with payloads."""
    for rows, cols, off in ((33, 37, 0), (129, 64, 1)):
        mat = _special_matrix(rows, cols, rows)
        flat = np.concatenate([np.zeros(off, np.float32), mat.reshape(-1)])
        got = _split_pack(lib, _cuda(flat), off, rows, cols, cols, transpose, b_role)
        _assert_bits(got, G.image(mat, transpose, b_role), (rows, cols, off))


@pytest.mark.parametrize("transpose", [False, True])
def test_split_pack_of_a_one_row_view(dev, transpose):
    """linear.split_pack of the transpose of an [n][1] column: a one-row view whose row stride is 1, not n.  The pack
    used to reject it as a leading dimension shorter than the row."""
    from distributed_rl_b200.linear import split_pack
    col = np.random.default_rng(5).standard_normal((129, 1)).astype(np.float32)
    x = _cuda(col).T
    assert x.shape == (1, 129) and x.stride(0) < 129
    for b_role in (False, True):
        _assert_bits(split_pack(x, transpose, b_role), G.image(col.T, transpose, b_role), b_role)


@pytest.mark.parametrize("rows", [(512, 512), (512, 512, 96), (256,)], ids=["apex", "stack_1120", "impala"])
def test_pack_pieces_matches_the_model(dev, rows):
    """The heads' piece layouts: stacked weights (forward B operand) and their transpose with the pieces side by side
    along the contraction (the W^T operand of dL/dx), written into a NaN-filled `out`."""
    from distributed_rl_b200.linear import _pack_pieces
    K = 2592 if rows == (256,) else 3136
    rng = np.random.default_rng(sum(rows))
    mats = [rng.standard_normal((r, K)).astype(np.float32) for r in rows]
    for transpose in (False, True):
        out = _filled(G.packed_floats(*((K, sum(rows)) if transpose else (sum(rows), K)), True))
        _pack_pieces([_cuda(m) for m in mats], transpose, True, out=out)
        _assert_bits(out, G.pieces_image(mats, transpose, True), (rows, transpose))


@pytest.mark.parametrize("C,HW", [(64, 49), (32, 81), (3, 7)], ids=["apex_r2d2", "impala", "k21"])
@pytest.mark.parametrize("transpose", [False, True])
def test_pack_act_nhwc_matches_the_model(lib, C, HW, transpose):
    """Both directions (transpose = 1 includes k_pack_zero_rows), ReLU on and off, batch sizes at the tile edges."""
    rng = np.random.default_rng(C * HW + int(transpose))
    for B in (1, 31, 32, 33, 127, 128, 129, 512, 1280):
        for relu in (1, 0):
            y = rng.standard_normal((B, HW, C)).astype(np.float32)
            rows, k = (C * HW, B) if transpose else (B, C * HW)
            out = _filled(G.packed_floats(rows, k, transpose))
            lib.check(lib.load().b2rl_gemm_pack_act_nhwc(_cuda(y).data_ptr(), B, HW, C, relu, int(transpose),
                                                          out.data_ptr(), _stream()))
            _assert_bits(out, G.act_image(y, bool(relu), transpose), (B, relu))


# k_rmsprop's image path: (piece rows, contraction, pieces that write images, centered, W^T image, early/late split)
_OPT_CASES = {
    "apex_centered_early": ((512, 512), 3136, (0, 1), True, True, True),
    "apex_plain_one": ((512, 512), 3136, (0, 1), False, True, False),
    "apex_second_only_no_wt": ((512, 512), 3136, (1,), True, False, False),
    "impala_plain_one": ((256,), 2592, (0,), False, True, False),
    "impala_centered_early_no_wt": ((256,), 2592, (0,), True, False, True),
    "stack_1120_centered_one": ((512, 512, 96), 3136, (1, 2), True, True, False),
    "stack_1120_plain_early": ((512, 512, 96), 3136, (0, 1, 2), False, True, True),
}


@pytest.mark.parametrize("case", list(_OPT_CASES), ids=list(_OPT_CASES))
def test_rmsprop_writes_the_images_of_the_new_weights(dev, case):
    """After each of two steps the rows of every updated piece in both images equal the model's image of its new
    weights; the rows of pieces that write no image and all padding keep their bits."""
    from distributed_rl_b200.linear import _pack_pieces
    from distributed_rl_b200.optim import FusedRMSprop
    rows, K, imaged, centered, with_wt, early = _OPT_CASES[case]
    total = sum(rows)
    g = torch.Generator(device="cuda")
    g.manual_seed(len(case))
    ws = [(torch.randn(r, K, device="cuda", generator=g) * 0.05).requires_grad_() for r in rows]
    other = (torch.randn(7, 33, device="cuda", generator=g)).requires_grad_()     # a tensor without images
    for w in ws + [other]:
        w.grad = torch.randn(w.shape, device="cuda", generator=g)
    params = [other] + ws
    opt = FusedRMSprop(params, lr=1e-3, alpha=0.95, eps=0.01, centered=centered)
    fwd = _filled(G.packed_floats(total, K, True))
    wt = _filled(G.packed_floats(K, total, True)) if with_wt else None
    with torch.no_grad():
        _pack_pieces(ws, False, True, out=fwd)
        if wt is not None:
            _pack_pieces(ws, True, True, out=wt)
    offs = np.cumsum((0,) + rows)[:-1]
    for i in imaged:
        opt.write_images(ws[i], fwd, wt, total, int(offs[i]))
    if early:
        assert opt.set_early([ws[i] for i in imaged])
    side = torch.cuda.Stream()
    held = [w.detach().cpu().numpy().copy() for w in ws]               # the rows the images hold
    for step in range(2):
        before = [w.detach().cpu().numpy().copy() for w in ws]
        if early:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                opt.step_early()
            torch.cuda.current_stream().wait_stream(side)
        opt.step()
        torch.cuda.synchronize()
        new = [w.detach().cpu().numpy() for w in ws]
        assert all(not np.array_equal(a, b) for a, b in zip(before, new))
        held = [new[i] if i in imaged else held[i] for i in range(len(ws))]
        _assert_bits(fwd, G.pieces_image(held, False, True), (case, step, "fwd"))
        if wt is not None:
            _assert_bits(wt, G.pieces_image(held, True, True), (case, step, "wt"))
        with torch.no_grad():
            for w in ws + [other]:
                w.grad.copy_(torch.randn(w.shape, device="cuda", generator=g))
        if early:
            assert opt.set_early([ws[i] for i in imaged])


# --------------------------------------------------------------------------------------------------------------------- #
# the GEMM, exact                                                                                                       #
# --------------------------------------------------------------------------------------------------------------------- #
def _three_term(a_np, b_np, k0=0, k1=None):
    """The fp64 3xTF32 product of A[:, k0:k1] and B[:, k0:k1] on the device."""
    a_hi, a_lo = G.split_tf32(a_np[:, k0:k1])
    b_hi, b_lo = G.split_tf32(b_np[:, k0:k1])
    d = lambda x: torch.from_numpy(x).cuda().double()       # noqa: E731
    return torch.cat([d(a_lo), d(a_hi), d(a_hi)], 1) @ torch.cat([d(b_hi), d(b_lo), d(b_hi)], 1).T


def _as_exact_fp32(ref64):
    ref = ref64.float()
    assert torch.equal(ref.double(), ref64), "the expected result is not representable in fp32"
    return ref


def _run_exact(lib, sms, a_img, b_img, a_np, b_np, M, N, K, ldc=None):
    """gemm_partials (through the C entry, into a sentinel-filled buffer with guard rows) and gemm_packed (into a
    guarded view) on the images of a_np and b_np: every partial and the result bit for bit, the guards unchanged.
    -> the half-chunk depths of the splits."""
    from distributed_rl_b200.linear import gemm_packed
    L = lib.load()
    if ldc is None:
        ldc = G.ceil_div(N, 4) * 4
    n_ws = L.b2rl_gemm_workspace_floats(M, N, K, ldc)
    n_splits = n_ws // (M * ldc) if n_ws else 1
    assert n_splits == G.splits(M, N, K, sms), (M, N, K, n_splits, sms)

    guard = 2 * ldc                                                      # two guard rows before and after
    buf = _filled(guard + n_splits * M * ldc + guard, SENTINEL_BITS)
    lib.check(L.b2rl_gemm_tf32x3_partials(a_img.data_ptr(), b_img.data_ptr(), buf.data_ptr() + 4 * guard,
                                          M, N, K, ldc, _stream()))
    parts = buf[guard:guard + n_splits * M * ldc].view(n_splits, M, ldc)
    sentinel = torch.tensor([SENTINEL_BITS], dtype=torch.int32, device="cuda")
    assert (buf[:guard].view(torch.int32) == sentinel).all() and (buf[-guard:].view(torch.int32) == sentinel).all()
    assert (parts[:, :, N:].view(torch.int32) == sentinel).all(), "a partial wrote past column N"
    for z in range(n_splits):
        c0, c1 = G.split_range(K, n_splits, z)
        want = _as_exact_fp32(_three_term(a_np, b_np, c0 * G.KC, min(c1 * G.KC, K)))
        assert torch.equal(parts[z, :, :N], want), f"{M}x{N}x{K}: partial {z} of {n_splits} (chunks {c0}..{c1})"
        del want

    ref = _as_exact_fp32(_three_term(a_np, b_np))
    cbuf = _filled((M + 2) * ldc, SENTINEL_BITS).view(M + 2, ldc)
    out = cbuf[1:M + 1, :N]
    got = gemm_packed(a_img, b_img, M, N, K, out=out)
    assert got.data_ptr() == out.data_ptr()
    assert torch.equal(out, ref), f"{M}x{N}x{K}: result ({n_splits} splits)"
    assert (cbuf[0].view(torch.int32) == sentinel).all() and (cbuf[M + 1].view(torch.int32) == sentinel).all()
    assert (cbuf[1:M + 1, N:].view(torch.int32) == sentinel).all(), "the result wrote past column N"
    del ref, cbuf, buf
    return G.depths(K, n_splits)


def _split_pack_t(x_np, transpose, b_role):
    from distributed_rl_b200.linear import split_pack
    return split_pack(_cuda(x_np), transpose, b_role)


def test_pipeline_depths(lib, sms):
    """144 output tiles: one split on this card, so K alone sets how many half-chunks the four-stage ring runs
    through, from two (it never wraps) to 64 (the 32-chunk cap)."""
    realised = {}
    for nk, K in G.DEPTH_K.items():
        a, b = G.exact_operands(G.DEPTH_M, G.DEPTH_N, K, seed=nk)
        d = _run_exact(lib, sms, _split_pack_t(a, False, False), _split_pack_t(b, False, True), a, b,
                       G.DEPTH_M, G.DEPTH_N, K)
        realised[nk] = d
    print("pipeline depths realised (nk per split):", realised)
    assert realised == {nk: [nk] for nk in G.DEPTH_K}, realised


def test_tile_edges(lib, sms):
    """M and N on both sides of the 128- and 256-row tiles, K at the chunk edges, ldc = ceil4(N) and wider."""
    seen = set()
    for M, N, K, ldc in G.edge_shapes():
        a, b = G.exact_operands(M, N, K, seed=M * 7 + N * 13 + K)
        # both operands through either transpose of split_pack
        t = (M + N) % 2 == 1
        a_img = _split_pack_t(np.ascontiguousarray(a.T) if t else a, t, False)
        b_img = _split_pack_t(b if t else np.ascontiguousarray(b.T), not t, True)
        d = _run_exact(lib, sms, a_img, b_img, a, b, M, N, K, ldc)
        seen.add((len(d), tuple(sorted(set(d)))))
    print("tile edges: (splits, nk) realised:", sorted(seen))


def _golden_shapes():
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_tf32x3_sm90.json")) as f:
        return json.load(f)["shapes"]


# the learners' producer of each recorded shape's operands
_PRODUCERS = {
    "apex_partials_512x1024x3136": ("act", "pieces"),            # heads forward: act image, stacked weights
    "apex_partials_1024x1024x3136": ("act", "pieces"),
    "apex_output_1024x3136x512": ("split_t", "act_t"),            # dL/dW: gh^T, x^T
    "apex_partials_512x3136x1024": ("split", "pieces_t"),         # dL/dx: gh, W^T (pieces side by side)
    "impala_output_256x2592x20480": ("split_t", "split_t"),
}


@pytest.mark.parametrize("entry", _golden_shapes(), ids=lambda e: e["name"])
def test_learner_shapes(lib, sms, entry):
    """The recorded shapes of the Ape-X, R2D2 and IMPALA learners with exact operands, each operand written by the
    producer the learner uses for it (split_pack otherwise)."""
    from distributed_rl_b200.linear import _pack_pieces
    M, N, K = entry["M"], entry["N"], entry["K"]
    pa, pb = _PRODUCERS.get(entry["name"], ("split", "split"))
    a, b = G.exact_operands(M, N, K, seed=entry["seed"], nonneg_a=pa == "act", nonneg_b=pb == "act_t")
    if pa == "act":                                              # A = flatten(relu(y)), y [M][49][64]
        x = G.relu_preimage(a, entry["seed"]).reshape(M, 64, 49).transpose(0, 2, 1)
        a_img = _filled(G.packed_floats(M, K, False))
        lib.check(lib.load().b2rl_gemm_pack_act_nhwc(_cuda(x).data_ptr(), M, 49, 64, 1, 0, a_img.data_ptr(),
                                                      _stream()))
    elif pa == "split_t":
        a_img = _split_pack_t(np.ascontiguousarray(a.T), True, False)
    else:
        a_img = _split_pack_t(a, False, False)
    if pb == "pieces":                                           # B = the stacked weights [N][K]
        b_img = _filled(G.packed_floats(N, K, True))
        _pack_pieces([_cuda(b[:N // 2]), _cuda(b[N // 2:])], False, True, out=b_img)
    elif pb == "pieces_t":                                       # B = W^T, W = [K][N] stacked from two pieces
        w = np.ascontiguousarray(b.T)
        b_img = _filled(G.packed_floats(N, K, True))
        _pack_pieces([_cuda(w[:K // 2]), _cuda(w[K // 2:])], True, True, out=b_img)
    elif pb == "act_t":                                          # B = x^T, x = flatten(relu(y)) [K][N], y [K][49][64]
        x = G.relu_preimage(np.ascontiguousarray(b.T), entry["seed"] + 1).reshape(K, 64, 49).transpose(0, 2, 1)
        b_img = _filled(G.packed_floats(N, K, True))
        lib.check(lib.load().b2rl_gemm_pack_act_nhwc(_cuda(x).data_ptr(), K, 49, 64, 1, 1, b_img.data_ptr(),
                                                      _stream()))
    elif pb == "split_t":
        b_img = _split_pack_t(np.ascontiguousarray(b.T), True, True)
    else:
        b_img = _split_pack_t(b, False, True)
    d = _run_exact(lib, sms, a_img, b_img, a, b, M, N, K)
    print(f"{entry['name']}: {len(d)} splits, nk {sorted(set(d))}")
