"""Fused gather + conv_1 (wgmma u8 x s8 with 4-digit weight split) against an fp64
convolution of the same inputs (torch CPU).  Floating-point kernel -> tolerance, stated
per assert; the contract is 1e-5."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import replay
    return replay


def _ref(frames_u8, w):
    x = torch.from_numpy(frames_u8).double() / 255.0
    return torch.nn.functional.conv2d(x, w.double().cpu(), stride=4)


@pytest.mark.parametrize("n_nets,n,relu", [(1, 1, False), (1, 5, False), (2, 37, True), (2, 300, False), (1, 512, True)])
def test_conv1_fused_matches_fp64_convolution(R, n_nets, n, relu):
    rng = np.random.default_rng(n * 10 + n_nets)
    rows = max(n, 8) + 11
    frames = rng.integers(0, 256, size=(rows, 4, 84, 84), dtype=np.uint8)
    frames[0, :, :8, :8] = 255                       # saturating corner
    idx = rng.integers(0, rows, size=n)
    idx[0] = 0
    ws = [torch.empty(32, 4, 8, 8).uniform_(-0.0625, 0.0625, generator=torch.Generator().manual_seed(7 + i))
          for i in range(n_nets)]
    ws[0][3] = 0.0                                   # an all-zero output channel
    ws[0][5, 0, 0, 0] = 0.9                          # one dominant weight: small digits of the others matter
    pack = R.Conv1Pack(n_nets, "cuda:0")
    for i, w in enumerate(ws):
        pack.pack(i, w.cuda())
    fr = torch.from_numpy(frames).cuda()
    outs = R.conv1_fused(fr, torch.from_numpy(idx).cuda(), pack, relu=relu)
    torch.cuda.synchronize()
    for i, (o, w) in enumerate(zip(outs, ws)):
        want = _ref(frames[idx], w)
        if relu:
            want = want.clamp_min(0)
        got = o.cpu().double()
        assert got.shape == want.shape == (n, 32, 20, 20)
        err = (got - want).abs().max().item()
        scale = want.abs().max().item()
        assert err <= 2e-6 * max(scale, 1.0), (i, err, scale)     # ~fp32 rounding of a 256-term sum
    # all rows in order when idx is None
    outs2 = R.conv1_fused(fr[:n].contiguous(), None, pack, relu=False)
    np.testing.assert_allclose(outs2[0].cpu().double().numpy(), _ref(frames[:n], ws[0]).numpy(), rtol=0, atol=2e-6 * 8)


@pytest.mark.parametrize("n_nets,n", [(1, 70), (2, 33)])
def test_conv1_fused_16_channels_impala(R, n_nets, n):
    """cfg/impala.json's conv_1 is 4 -> 16 channels: same kernel, C_OUT = 16 instantiation."""
    rng = np.random.default_rng(n)
    frames = rng.integers(0, 256, size=(n, 4, 84, 84), dtype=np.uint8)
    ws = [torch.empty(16, 4, 8, 8).uniform_(-0.0625, 0.0625, generator=torch.Generator().manual_seed(3 + i))
          for i in range(n_nets)]
    pack = R.Conv1Pack(n_nets, "cuda:0", c_out=16)
    for i, w in enumerate(ws):
        pack.pack(i, w.cuda())
    outs = R.conv1_fused(torch.from_numpy(frames).cuda(), None, pack, relu=True)
    for o, w in zip(outs, ws):
        want = _ref(frames, w).clamp_min(0)
        assert o.shape == (n, 16, 20, 20)
        assert (o.cpu().double() - want).abs().max().item() <= 2e-6 * max(want.abs().max().item(), 1.0)


def test_conv1_fused_reads_replay_field_in_place(R):
    """Gather fused: rows come straight from the DeviceReplay payload (no staging copy)."""
    from oracle import oracle as O
    cap = 256
    rep = R.DeviceReplay(cap, fields=R.APEX_FIELDS)
    rep.fill_hash(cap, seed=3)
    rep.build(torch.rand(cap, device="cuda") + 0.1)
    idx, _, _ = rep.sample(64)
    w = torch.empty(32, 4, 8, 8).uniform_(-0.06, 0.06, generator=torch.Generator().manual_seed(1))
    pack = R.Conv1Pack(1, "cuda:0"); pack.pack(0, w.cuda())
    out = R.conv1_fused(rep.field_view("next_state"), idx, pack)[0]
    frames = O.hash_rows(1, idx.cpu().numpy(), R.FRAME_STACK_BYTES, 3).reshape(-1, 4, 84, 84)
    want = _ref(frames, w)
    assert (out.cpu().double() - want).abs().max().item() <= 2e-6 * max(want.abs().max().item(), 1.0)
    rep.close()


def _wgrad_ref(frames_u8, idx, gy):
    x = (torch.from_numpy(frames_u8[idx]).double() / 255.0)
    return torch.nn.grad.conv2d_weight(x, (gy.shape[1], 4, 8, 8), gy.double().cpu(), stride=4)


@pytest.mark.parametrize("c_out,n", [(32, 1), (32, 5), (32, 300), (16, 37), (32, 512), (16, 600)])
def test_conv1_wgrad_matches_fp64(R, c_out, n):
    """Fused gather + conv_1 weight gradient (csrc/conv1_wgrad.cu) against an fp64 wgrad of the same rows.
    Tolerance: 2e-6 of the largest |dW| entry (exact integer accumulation of 28-bit fixed-point gy;
    the only roundings are the digit truncation at 2^-29 of the channel max and the final fp32 store)."""
    rng = np.random.default_rng(n + c_out)
    rows = max(n, 8) + 7
    frames = rng.integers(0, 256, size=(rows, 4, 84, 84), dtype=np.uint8)
    frames[1] = 255
    idx = rng.integers(0, rows, size=n)
    idx[0] = 1
    g = torch.Generator().manual_seed(n)
    gy = torch.randn(n, c_out, 20, 20, generator=g) * torch.logspace(-6, 0, n).view(n, 1, 1, 1)   # wide range over items
    gy[:, 3] = 0.0                                    # an all-zero channel
    gy[0, 5, 0, 0] = 50.0                             # one dominant entry
    gy = gy * (torch.rand(n, c_out, 20, 20, generator=g) > 0.5)   # ReLU-masked, like the real dL/dy
    gyc = gy.cuda().contiguous(memory_format=torch.channels_last)
    fr = torch.from_numpy(frames).cuda()
    gw = R.conv1_wgrad(fr, torch.from_numpy(idx).cuda(), gyc)
    ref = _wgrad_ref(frames, idx, gy)
    assert gw.shape == (c_out, 4, 8, 8)
    err = (gw.double().cpu() - ref).abs().max().item()
    assert err <= 2e-6 * ref.abs().max().item(), (err, ref.abs().max().item())
    assert (gw[3] == 0).all()
    # idx=None takes rows 0..n-1; accumulate adds into an existing gradient
    gw2 = R.conv1_wgrad(fr[:n].contiguous(), None, gyc)
    ref2 = _wgrad_ref(frames, np.arange(n), gy)
    assert (gw2.double().cpu() - ref2).abs().max().item() <= 2e-6 * ref2.abs().max().item()
    acc = gw2.clone()
    R.conv1_wgrad(fr[:n].contiguous(), None, gyc, out=acc, accumulate=True)
    torch.testing.assert_close(acc, 2 * gw2, rtol=1e-6, atol=0)
    # deterministic
    assert torch.equal(R.conv1_wgrad(fr, torch.from_numpy(idx).cuda(), gyc), gw)
    # ReLU mask of the fused forward: gy * (y > 0) applied inside the kernel
    yk = torch.relu(torch.randn(n, c_out, 20, 20, generator=g))
    gwm = R.conv1_wgrad(fr, torch.from_numpy(idx).cuda(), gyc,
                        relu_y=yk.cuda().contiguous(memory_format=torch.channels_last))
    refm = _wgrad_ref(frames, idx, gy * (yk > 0))
    assert (gwm.double().cpu() - refm).abs().max().item() <= 2e-6 * max(refm.abs().max().item(), 1e-30)
