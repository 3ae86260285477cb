"""GPU tests of the dense heads' resident operand images (the fused optimizer keeps the online ones current, a target
sync or a state-dict load repacks them) and of the dL/dx split-K partials summed by the unflatten + ReLU-mask kernel."""
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture(autouse=True)
def _deterministic():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def _mk(early=True, seed=0, B=64, N=8192):
    from distributed_rl_b200 import apex
    cfg = apex.ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                          CUDNN_BENCHMARK=False, EARLY_HEAD_UPDATE=early)
    torch.manual_seed(seed)
    L = apex.Learner(cfg, connect=None, start_replay=False)
    with torch.no_grad():
        for p in L.target_model.parameters():
            p.add_(0.01 * torch.randn(p.shape, device=p.device))
    st = L.memory.store
    st.fill_hash(N, seed=1)
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    st.field_view("action").copy_(torch.randint(0, 6, (N,), device="cuda", generator=g, dtype=torch.int32))
    st.field_view("reward").copy_(torch.randn(N, device="cuda", generator=g).clamp_(-1, 1))
    st.field_view("done").copy_((torch.rand(N, device="cuda", generator=g) < 0.1).to(torch.uint8))
    st.build((torch.randn(N, device="cuda", generator=g).abs().clamp(max=1) + 1e-7) ** 0.6)
    st.seed(99, 0)
    return L


def _assert_images_current(model, want_bwdT):
    from distributed_rl_b200.linear import _pack_pieces
    pieces = model.head_pieces()
    assert pieces and model._resident
    for group, ws in pieces:
        imgs = model._resident[group]
        assert set(imgs) == ({"fwd", "bwdT"} if want_bwdT else {"fwd"})
        for k, img in imgs.items():
            assert torch.equal(img, _pack_pieces(ws, k == "bwdT", True)), k


@pytest.mark.parametrize("early", [True, False])
def test_resident_images_follow_the_weights_through_captured_steps(early):
    L = _mk(early=early)
    for _ in range(3):
        L.fused_step(use_graph=True)
    torch.cuda.synchronize()
    assert L._fused.resident is not None
    _assert_images_current(L.model, True)
    _assert_images_current(L.target_model, False)


def test_target_sync_and_state_dict_load_refresh_the_images():
    """After a target sync and a load_state_dict into the online model between replays, the next step equals that of
    a learner built fresh with the same weights, tree and draw, bit for bit."""
    L = _mk(seed=0)
    for _ in range(2):
        L.fused_step(use_graph=True)
    torch.manual_seed(7)
    new_online = {k: v + 0.01 * torch.randn_like(v) for k, v in L.model.state_dict().items()}
    L.target_model.updateParameter(L.model, 1)
    L.model.load_state_dict(new_online)
    torch.cuda.synchronize()
    _assert_images_current(L.model, True)
    _assert_images_current(L.target_model, False)

    F = _mk(seed=1)
    F.model.load_state_dict(L.model.state_dict())
    F.target_model.load_state_dict(L.target_model.state_dict())
    for a, b in zip(F.optim.square_avg + F.optim.grad_avg, L.optim.square_avg + L.optim.grad_avg):
        a.copy_(b)
    F.memory.store.build(L.memory.store.priorities().clone())
    F.memory.store.seed(123, 0)
    L.memory.store.seed(123, 0)
    outs = []
    for learner, graph in ((L, True), (F, False)):     # L replays its graph; F runs the same step once, eagerly
        out = learner.fused_step(use_graph=graph)
        torch.cuda.synchronize()
        outs.append((out["idx"].clone(), out["prio"].clone(), out["scalars"].clone(),
                     [p.detach().clone() for p in learner.model.parameters()]))
    (i0, p0, s0, w0), (i1, p1, s1, w1) = outs
    assert torch.equal(i0, i1)
    assert torch.equal(p0, p1)
    assert torch.equal(s0, s1)
    for a, b in zip(w0, w1):
        assert torch.equal(a, b)


@pytest.mark.parametrize("splits", [1, 2, 4, 8])
def test_unflatten_sums_split_partials_in_order(splits):
    """k_unflatten_relu_mask over `splits` partials == the partials summed left to right (what k_splitk_reduce
    does), then the plain kernel; at the step's shape (B = 512, 64 x 7 x 7)."""
    from distributed_rl_b200 import _lib
    from distributed_rl_b200.linear import _stream
    B, C, HW = 512, 64, 49
    K = C * HW
    g = torch.Generator(device="cuda"); g.manual_seed(splits)
    part = torch.randn(splits, B, K, device="cuda", generator=g)
    y = torch.randn(B, HW, C, device="cuda", generator=g)
    summed = part[0].clone()
    for z in range(1, splits):
        summed += part[z]
    L = _lib.load()
    got = torch.empty_like(y)
    want = torch.empty_like(y)
    _lib.check(L.b2rl_unflatten_relu_mask(part.data_ptr(), K, splits, B * K, y.data_ptr(), B, HW, C, got.data_ptr(),
                                          _stream()))
    _lib.check(L.b2rl_unflatten_relu_mask(summed.data_ptr(), K, 1, 0, y.data_ptr(), B, HW, C, want.data_ptr(),
                                          _stream()))
    ref = torch.where(y > 0, summed.view(B, C, HW).transpose(1, 2), torch.zeros_like(y))
    assert torch.equal(got, want)
    assert torch.equal(want, ref)


def test_gemm_partials_sum_to_the_reduced_gemm():
    """b2rl_gemm_tf32x3_partials summed in split order == b2rl_gemm_tf32x3 at the heads' dL/dx shape."""
    from distributed_rl_b200.linear import gemm_packed, gemm_partials, split_pack
    M, N, K = 512, 3136, 1024
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(K, N, device="cuda", generator=g)
    pa, pb = split_pack(a, False, False), split_pack(w, True, True)
    want = gemm_packed(pa, pb, M, N, K)
    part, splits, ldc = gemm_partials(pa, pb, M, N, K)
    part = part.view(splits, M, ldc)
    got = part[0].clone()
    for z in range(1, splits):
        got += part[z]
    assert torch.equal(got[:, :N], want)


@pytest.mark.parametrize("M,splits", [(1024, 4), (512, 8), (512, 2), (1000, 3)])
def test_dueling_forward_sums_split_partials_in_order(M, splits):
    """k_dueling_forward over `splits` partials of h == the partials summed left to right (k_splitk_reduce), then
    the plain kernel: q and the summed h bit for bit, at the step's shapes (2H = 1024, A = 6) and a ragged M."""
    from distributed_rl_b200 import _lib
    from distributed_rl_b200.linear import _stream
    H, A = 512, 6
    g = torch.Generator(device="cuda"); g.manual_seed(M + splits)
    part = torch.randn(splits, M, 2 * H, device="cuda", generator=g)
    wa = torch.randn(A, H, device="cuda", generator=g) * 0.05
    wv = torch.randn(1, H, device="cuda", generator=g) * 0.05
    summed = part[0].clone()
    for z in range(1, splits):
        summed += part[z]
    L = _lib.load()
    q_got, q_want = torch.empty(M, A, device="cuda"), torch.empty(M, A, device="cuda")
    h_got = torch.empty(M, 2 * H, device="cuda")
    _lib.check(L.b2rl_dueling_forward(part.data_ptr(), splits, M * 2 * H, M, H, wa.data_ptr(), A, wv.data_ptr(),
                                      q_got.data_ptr(), h_got.data_ptr(), _stream()))
    _lib.check(L.b2rl_dueling_forward(summed.data_ptr(), 1, 0, M, H, wa.data_ptr(), A, wv.data_ptr(),
                                      q_want.data_ptr(), None, _stream()))
    assert torch.equal(h_got, summed)
    assert torch.equal(q_got, q_want)
    r = summed.double().clamp_min(0)
    adv = r[:, :H] @ wa.double().T
    ref = adv + r[:, H:] @ wv.double().T - adv.mean(1, keepdim=True)
    assert (q_want.double() - ref).abs().max() < 1e-4
