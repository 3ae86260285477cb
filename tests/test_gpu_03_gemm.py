"""3xTF32 dense layer (csrc/gemm.cu, wgmma tf32) against an fp64 matmul of the same inputs.
Floating-point kernel -> tolerance, stated per assert: the error must be of the order of an fp32
FMA chain (the cuBLAS fp32 SIMT GEMM the reference's nn.Linear runs as), far below plain TF32."""
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import linear
    return linear


def _rel(a, ref):
    return ((a.double() - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize("M,N,K", [(512, 1024, 3136), (512, 512, 3136), (1, 6, 512), (37, 19, 100), (130, 300, 33),
                                   (512, 3136, 1024), (1024, 3136, 512)])
def test_forward_matches_fp64(L, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) * 0.05
    x[0, 0] = 1e4                                      # wide dynamic range within a row
    ref = x.double() @ w.double().T
    y = L.linear3x(x, w)
    assert y.shape == (M, N)
    e3, e32 = _rel(y, ref), _rel(x @ w.T, ref)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        e_tf32 = _rel(x @ w.T, ref)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    assert e3 < 5e-6, (e3, e32, e_tf32)                # fp32-class accuracy
    assert e3 < 4 * e32 + 5e-7, (e3, e32, e_tf32)      # per-product error 2^-22 (dropped lo*lo, TF32-truncated lo) + tensor-core accumulation
    if K >= 512 and M > 1:
        assert e3 < e_tf32 / 20, (e3, e32, e_tf32)     # ... and far from what plain TF32 gives


def test_backward_matches_fp64(L):
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(512, 3136, device="cuda", generator=g, requires_grad=True)
    w = (torch.randn(1024, 3136, device="cuda", generator=g) * 0.02).requires_grad_()
    gy = torch.randn(512, 1024, device="cuda", generator=g)
    L.linear3x(x, w).backward(gy)
    gx_ref = gy.double() @ w.detach().double()
    gw_ref = gy.double().T @ x.detach().double()
    assert _rel(x.grad, gx_ref) < 5e-6
    assert _rel(w.grad, gw_ref) < 5e-6


def test_odd_shapes_backward(L):
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(37, 100, device="cuda", generator=g, requires_grad=True)
    w = torch.randn(19, 100, device="cuda", generator=g, requires_grad=True)
    y = L.linear3x(x, w)
    y.square().sum().backward()
    xr = x.detach().double().requires_grad_()
    wr = w.detach().double().requires_grad_()
    (xr @ wr.T).square().sum().backward()
    assert _rel(y, (xr @ wr.T).detach()) < 5e-6
    assert _rel(x.grad, xr.grad) < 5e-6
    assert _rel(w.grad, wr.grad) < 5e-6


def test_special_values_do_not_leak(L):
    x = torch.zeros(4, 32, device="cuda")
    w = torch.zeros(8, 32, device="cuda")
    x[1, 3] = float("inf")
    w[2, 3] = 1.0
    x[2, 5] = 3e-39                                    # subnormal input: flushed or kept, never NaN
    w[:, 5] = 1.0
    y = L.linear3x(x, w)
    assert not torch.isfinite(y[1, 2])                 # inf input: non-finite output (inf*0 of the lo term -> NaN)
    assert torch.isfinite(y[0]).all() and torch.isfinite(y[2]).all() and torch.isfinite(y[3]).all()


def test_stacked_weights_and_cache(L):
    """Sibling heads: two weights sharing the input, packed into one operand without a cat; the packed
    forward operand can be cached across passes; gradients reach each weight."""
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(64, 3136, device="cuda", generator=g, requires_grad=True)
    w1 = (torch.randn(512, 3136, device="cuda", generator=g) * 0.02).requires_grad_()
    w2 = (torch.randn(70, 3136, device="cuda", generator=g) * 0.02).requires_grad_()
    cache = {}
    y = L.linear3x(x, [w1, w2], cache)
    y2 = L.linear3x(x.detach(), [w1, w2], cache)          # served from the cached operand
    assert torch.equal(y.detach(), y2) and "fwd" in cache
    ref = x.detach().double() @ torch.cat([w1, w2]).detach().double().T
    assert _rel(y, ref) < 5e-6
    gy = torch.randn(64, 582, device="cuda", generator=g)
    y.backward(gy)
    assert _rel(x.grad, gy.double() @ torch.cat([w1, w2]).detach().double()) < 5e-6
    gw = gy.double().T @ x.detach().double()
    assert _rel(w1.grad, gw[:512]) < 5e-6 and _rel(w2.grad, gw[512:]) < 5e-6
    # a non-32-multiple inner piece falls back to one concatenated operand
    y3 = L.linear3x(x.detach(), [w2.detach(), w1.detach()])
    assert _rel(y3, x.detach().double() @ torch.cat([w2, w1]).detach().double().T) < 5e-6


@pytest.mark.parametrize("M,H,A", [(512, 512, 6), (1, 32, 1), (37, 96, 18), (64, 1024, 32), (3840, 512, 6)])
def test_dueling_tail_matches_pytorch(L, M, H, A):
    """csrc/dueling.cu against the unfused node sequence (ReLU, two Linear, Add, Mean, Substract) in fp64."""
    g = torch.Generator(device="cuda").manual_seed(M + H + A)
    h = torch.randn(M, 2 * H, device="cuda", generator=g).requires_grad_()
    wa = (torch.randn(A, H, device="cuda", generator=g) * 0.05).requires_grad_()
    wv = (torch.randn(1, H, device="cuda", generator=g) * 0.05).requires_grad_()
    gq = torch.randn(M, A, device="cuda", generator=g)
    assert L.dueling_tail_supported(h, wa, wv)
    q = L.dueling_tail(h, wa, wv)
    q.backward(gq)
    hd, wad, wvd = (t.detach().double().requires_grad_() for t in (h, wa, wv))
    r = torch.relu(hd)
    adv, val = r[:, :H] @ wad.T, r[:, H:] @ wvd.T
    qr = (adv + val) - adv.mean(dim=-1, keepdim=True)
    qr.backward(gq.double())
    for got, ref in ((q, qr.detach()), (h.grad, hd.grad), (wa.grad, wad.grad), (wv.grad, wvd.grad)):
        assert (got.double() - ref).abs().max().item() <= 2e-6 * max(ref.abs().max().item(), 1e-3)
    # deterministic
    h2 = h.detach().clone().requires_grad_()
    L.dueling_tail(h2, wa, wv).backward(gq)
    assert torch.equal(h2.grad, h.grad)


def test_graph_agent_fused_tail_equals_node_sequence():
    """GraphAgent with the fused first layer (3xTF32) + fused dueling tail == the plain node-by-node graph."""
    from distributed_rl_b200.agent import GraphAgent
    from distributed_rl_b200.apex import default_apex_model
    torch.manual_seed(0)
    m = GraphAgent(default_apex_model()).cuda()
    x = torch.rand(48, 4, 84, 84, device="cuda")
    outs, grads = [], []
    for fused in (False, True):
        m.fused_dueling_tail = m.dense_3xtf32 = fused
        m.zero_grad(set_to_none=True)
        q = m([x])[0]
        q.square().sum().backward()
        outs.append(q.detach().clone())
        grads.append([p.grad.clone() for p in m.parameters()])
    torch.testing.assert_close(outs[1], outs[0], rtol=1e-4, atol=1e-5)
    for a, b in zip(grads[1], grads[0]):
        torch.testing.assert_close(a, b, rtol=2e-3, atol=1e-4 * b.abs().max().item())


def test_relu_flatten_folded_into_the_packs_matches_fp64(L):
    """linear.relu_flat_linear3x: h = flatten_NCHW(relu(y)) @ W^T read straight from the conv stack's channels_last
    output (ReLU applied while packing, the NHWC <-> NCHW feature permutation carried by the weight / x^T packs,
    csrc/gemm.cu colmap) against act + nn.Flatten + matmul in fp64 — forward, dL/dy (with the ReLU mask) and dL/dW."""
    g = torch.Generator(device="cuda").manual_seed(11)
    B, C, H, W = 96, 64, 7, 7
    y = torch.randn(B, C, H, W, device="cuda", generator=g).contiguous(memory_format=torch.channels_last).requires_grad_()
    w1 = (torch.randn(512, C * H * W, device="cuda", generator=g) * 0.02).requires_grad_()
    w2 = (torch.randn(512, C * H * W, device="cuda", generator=g) * 0.02).requires_grad_()
    gh = torch.randn(B, 1024, device="cuda", generator=g)
    assert L.relu_flat_supported(y, [w1, w2])
    h = L.relu_flat_linear3x(y, [w1, w2])
    h.backward(gh)
    yd = y.detach().double().requires_grad_()
    wd = torch.cat([w1, w2]).detach().double().requires_grad_()
    href = torch.relu(yd).flatten(1) @ wd.T                      # nn.Flatten of the logical NCHW tensor
    href.backward(gh.double())
    assert _rel(h, href.detach()) < 5e-6
    assert y.grad.shape == y.shape and y.grad.is_contiguous(memory_format=torch.channels_last)
    assert _rel(y.grad, yd.grad) < 5e-6
    assert _rel(torch.cat([w1.grad, w2.grad]), wd.grad) < 5e-6
    assert (y.grad[y.detach() <= 0] == 0).all()                  # ReLU mask applied

