"""CPU tests of the IMPALA residual network (netCat RESCNN2D, impala.resnet_small_model): the node's layers, feature
sizes and parameter count, the config round trip, the refusals that need no GPU, the numpy restatement of the
fused stem's arithmetic (tests/stem_model.py) at a tiny size against float64, and its torch restatement against the
numpy one."""
import os
import sys
import types

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import stem_model as M  # noqa: E402


def test_the_node_is_the_papers_large_network_without_its_lstm():
    from distributed_rl_b200 import impala
    from distributed_rl_b200.agent import GraphAgent, ResidualBlock
    net = GraphAgent(impala.resnet_small_model())
    stack = net.module00
    names = [n for n, _ in stack.named_children()]
    want = []
    for i in (1, 2, 3):
        want += [f"conv_{i}", f"pool_{i}", f"block_{i}_1", f"block_{i}_2"]
    assert names == want + ["act", "Flatten"]
    for i, (cin, cout) in enumerate(((4, 16), (16, 32), (32, 32)), 1):
        c = getattr(stack, f"conv_{i}")
        assert (c.in_channels, c.out_channels, c.kernel_size, c.stride, c.padding, c.bias) == \
            (cin, cout, (3, 3), (1, 1), (1, 1), None)
        p = getattr(stack, f"pool_{i}")
        assert (p.kernel_size, p.stride, p.padding) == (3, 2, 1)
        for j in (1, 2):
            b = getattr(stack, f"block_{i}_{j}")
            assert isinstance(b, ResidualBlock)
            for c in (b.conv_1, b.conv_2):
                assert (c.in_channels, c.out_channels, c.kernel_size, c.padding, c.bias) == (cout, cout, (3, 3), (1, 1), None)
    x = torch.rand(2, 4, 84, 84)
    sizes = []
    h = x
    for name, layer in stack.named_children():
        h = layer(h)
        if name.startswith("pool_"):
            sizes.append(h.shape[-1])
    assert sizes == [42, 21, 11] and h.shape == (2, 3872)
    assert sum(p.numel() for p in net.parameters()) == 1_090_368
    assert net.forward([x])[0].shape == (2, 7)
    assert net.first_stem_node() == "module00" and net.first_conv_node() is None
    # the forward from the stem's pooled output is the forward
    pooled = stack.pool_1(stack.conv_1(x))
    torch.testing.assert_close(net.forward_from_stem(pooled)[0], net.forward([x])[0], rtol=0, atol=0)
    sd = net.state_dict()
    assert "module00.conv_1.weight" in sd and "module00.block_3_2.conv_2.weight" in sd and "module01.MLP_1.weight" in sd


def test_a_stem_the_kernels_do_not_run_is_not_named():
    from distributed_rl_b200 import impala
    from distributed_rl_b200.agent import GraphAgent
    m = impala.resnet_small_model()
    m["module00"]["nUnit"] = [32, 32, 32]
    m["module01"]["iSize"] = 32 * 11 * 11
    assert GraphAgent(m).first_stem_node() is None
    with pytest.raises(ValueError, match="RESCONV2D"):
        GraphAgent({"m": {"netCat": "RESCONV2D", "iSize": 4, "prior": 0, "input": [0], "output": True}})


def test_the_config_round_trip_through_from_configuration(monkeypatch):
    from distributed_rl_b200 import impala
    cfg = types.ModuleType("configuration")
    defaults = impala.ImpalaConfig()
    for k in ("BATCHSIZE", "ACTION_SIZE", "GAMMA", "C_LAMBDA", "C_VALUE", "P_VALUE", "ENTROPY_R", "UNROLL_STEP",
              "REPLAY_MEMORY_LEN", "BUFFER_SIZE", "LEARNER_DEVICE", "REDIS_SERVER", "OPTIM_INFO"):
        setattr(cfg, k, getattr(defaults, k))
    cfg.MODEL = impala.resnet_small_model()
    cfg.LEARNER_DEVICE = "cpu"
    monkeypatch.setitem(sys.modules, "configuration", cfg)
    c = impala.ImpalaConfig.from_configuration()
    assert c.MODEL == impala.resnet_small_model() and c.FUSED_CONV1 and c.DENSE_3XTF32
    assert c == impala.ImpalaConfig(MODEL=impala.resnet_small_model(), LEARNER_DEVICE="cpu")


def test_the_learner_refuses_a_captured_step_without_a_fused_first_layer():
    from distributed_rl_b200 import impala
    m = impala.resnet_small_model()
    m["module00"]["nUnit"] = [32, 32, 32]
    m["module01"]["iSize"] = 32 * 11 * 11
    L = types.SimpleNamespace(model=__import__("distributed_rl_b200.agent", fromlist=["GraphAgent"]).GraphAgent(m),
                              cfg=impala.ImpalaConfig(), device=torch.device("cpu"))
    with pytest.raises(ValueError, match="RESCNN2D stem"):
        impala._DrawnRollouts(L)
    with pytest.raises(ValueError, match="RESCNN2D stem"):
        impala._BoundRollouts(L)


def _frames(n, H, seed):
    """Random stacks, constant stacks and stacks of flat blocks (exact ties inside and across windows)."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, size=(n, 4, H, H), dtype=np.uint8)
    f[1] = 0
    f[2] = 200
    blocks = rng.integers(0, 256, size=(4, (H + 2) // 3, (H + 2) // 3), dtype=np.uint8)
    f[3] = np.repeat(np.repeat(blocks, 3, axis=1), 3, axis=2)[:, :H, :H]
    return f


def test_the_digits_reconstruct_the_weights():
    w = np.random.default_rng(0).standard_normal((16, 4, 3, 3)).astype(np.float32) * 0.1
    w[5] = 0.0
    q, scale = M.pack(w)
    assert np.abs(q).max() <= 127
    m = np.abs(w.reshape(16, -1)).max(axis=1)
    s = np.where(m > 0, m / np.float32(127), np.float32(1)).astype(np.float32)
    assert np.array_equal(scale, s / np.float32(255))        # the kernel's scale: the /255 folded in
    rec = (q[0] + q[1] / 2 ** 7 + q[2] / 2 ** 14 + q[3] / 2 ** 21) * s.astype(np.float64)[:, None]
    err = np.abs(rec - w.reshape(16, -1)).max(axis=1)
    assert np.all(err <= s * 2.0 ** -22)
    assert not rec[5].any()


@pytest.mark.parametrize("H", [9, 10])
def test_the_stem_model_against_float64(H):
    """The forward within conv_1's bound of an fp64 conv + max-pool; the argmax is torch's max_pool2d index on the
    model's own values (the first maximum: exact ties are common); the folded pool backward is torch's max-pool
    backward; the weight gradient is within 2e-6 of the largest |dW| of an fp64 one routed through that argmax."""
    F = torch.nn.functional
    n = 5
    frames = _frames(n, H, seed=H)
    w = np.random.default_rng(1).standard_normal((16, 4, 3, 3)).astype(np.float32) * 0.1
    y = M.conv(frames, w)
    x64 = torch.from_numpy(frames).double() / 255
    y64 = F.conv2d(x64, torch.from_numpy(w).double(), padding=1)
    assert np.abs(y - y64.numpy()).max() <= 2e-6 * np.abs(y64.numpy()).max()
    pooled, arg = M.pool(y)
    p64 = F.max_pool2d(y64, 3, 2, 1)
    assert np.abs(pooled - p64.numpy()).max() <= 2e-6 * np.abs(p64.numpy()).max()
    yt = torch.from_numpy(y).double().requires_grad_(True)
    pt, it = F.max_pool2d(yt, 3, 2, 1, return_indices=True)
    assert np.array_equal(pooled, pt.detach().numpy().astype(np.float32))
    PH = pooled.shape[-1]
    py, px = np.meshgrid(np.arange(PH), np.arange(PH), indexing="ij")
    iy, ix = it.numpy() // H, it.numpy() % H
    assert np.array_equal(arg, (3 * (iy - 2 * py + 1) + (ix - 2 * px + 1)).astype(np.uint8))
    assert (arg[1] != arg[1].flat[0]).any() or PH == 1          # constant stacks: the borders pick other positions
    assert arg[1, :, 1:, 1:].max() == 0 and arg[1, :, 0, 1:].min() == 3    # first valid position of a tied window
    gp = np.random.default_rng(2).standard_normal(pooled.shape).astype(np.float32)
    pt.backward(torch.from_numpy(gp).double())
    g = M.fold(gp, arg, H, H, np.float64)
    assert np.array_equal(g, yt.grad.numpy())
    g32 = M.fold(gp, arg, H, H)
    assert np.abs(g32 - g).max() <= 2 ** -22 * np.abs(g).max()
    dw = M.wgrad(frames, gp, arg)
    dw64 = torch.nn.grad.conv2d_weight(x64, (16, 4, 3, 3), torch.from_numpy(g), padding=1).numpy().reshape(16, 36)
    assert np.abs(dw - dw64).max() <= 2e-6 * np.abs(dw64).max()


def test_the_stem_entry_points_refuse_bad_arguments_before_any_launch():
    """Null pointers, a coded frame pool and an Ape-X plane table are refused on the host (no device needed)."""
    import ctypes as C
    from distributed_rl_b200 import _lib
    try:
        lib = _lib.load()
    except _lib.B2RLError:
        pytest.skip("libb2rl.so is not built")
    n0 = lib.b2rl_launch_count()
    dummy = C.c_void_p(16)
    coded = _lib.Frames(pool=16, planes=16, offsets=16, pool_units=1, pool_frames=1, rows=1)
    apex = _lib.Frames(pool=16, planes=16, plane_stride=8, rows=1)
    apex0 = _lib.Frames(pool=16, planes=16, plane_stride=0, plane_base=4, rows=1)
    stacks = _lib.Frames(base=16, row_stride=28224, rows=1)
    for f, msg in ((coded, b"coded"), (apex, b"plane_stride 8"), (apex0, b"plane_stride 8")):
        assert lib.b2rl_stem_fused(f, None, 1, dummy, dummy, dummy, dummy, None) == -1
        assert msg in lib.b2rl_last_error()
        assert lib.b2rl_stem_wgrad(f, None, 1, dummy, dummy, dummy, dummy, 0, None) == -1
        assert msg in lib.b2rl_last_error()
    assert lib.b2rl_stem_fused(stacks, None, 1, None, dummy, dummy, dummy, None) == -1
    assert lib.b2rl_stem_wgrad(stacks, None, 0, dummy, dummy, dummy, dummy, 0, None) == -1
    assert lib.b2rl_stem_wgrad(stacks, None, 1, C.c_void_p(20), dummy, dummy, dummy, 0, None) == -1
    assert b"16-byte" in lib.b2rl_last_error()
    assert lib.b2rl_stem_pack(None, dummy, dummy, None) == -1
    assert lib.b2rl_launch_count() == n0


def _edge_stacks(n, H, seed):
    """n >= 7 stacks: random, constant 0, 255 and 77, flat 3x3 and 4x4 blocks (exact ties inside and across
    windows), and random again."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, size=(n, 4, H, H), dtype=np.uint8)
    f[1], f[2], f[3] = 0, 255, 77
    for k, b in ((4, 3), (5, 4)):
        blocks = rng.integers(0, 256, size=(4, (H + b - 1) // b, (H + b - 1) // b), dtype=np.uint8)
        f[k] = np.repeat(np.repeat(blocks, b, axis=1), b, axis=2)[:, :H, :H]
    return f


@pytest.mark.parametrize("H", [9, 10, 84])
def test_the_torch_restatement_is_the_numpy_model(H):
    """stem_model's torch functions (which the GPU tests run at 21 504 stacks) against its numpy loops: the forward's
    pooled values and argmax bit for bit, in chunks and through a permuting, repeating idx; the fold bit for bit in
    fp32 and fp64; the weight gradient within one fp32 ulp (the two sum the stacks in other float64 orders), with
    stacks of small gradients (their own digit scale) and of gradients so small the digit exponent clamps at 27."""
    n = 7
    frames = _edge_stacks(n, H, seed=H)
    w = np.random.default_rng(3).standard_normal((16, 4, 3, 3)).astype(np.float32) * 0.1
    w[2] = 0.0
    w[6, 1, 1, 1] = 2.0                                     # one dominant weight: the small ones live in the low digits
    want_p, want_a = M.pool(M.conv(frames, w))
    ft, wt = torch.from_numpy(frames), torch.from_numpy(w)
    got_p, got_a = M.forward_t(ft, None, wt, chunk=3)
    assert np.array_equal(got_p.numpy().view(np.uint32), want_p.view(np.uint32))
    assert np.array_equal(got_a.numpy(), want_a)
    idx = torch.tensor([6, 0, 4, 4, 1, 5, 2, 3, 0])
    p_i, a_i = M.forward_t(ft, idx, wt, chunk=4)
    assert torch.equal(p_i, got_p[idx]) and torch.equal(a_i, got_a[idx])

    rng = np.random.default_rng(4)
    gp = rng.standard_normal(want_p.shape).astype(np.float32)
    gp[3] *= np.float32(1e-3)
    gp[4] *= np.float32(1e-33)                               # 4 max|gp| / 127 below 2^-100: the exponent clamps
    gp[5] = np.abs(gp[5]) * np.exp2(-rng.uniform(0, 30, size=gp[5].shape)).astype(np.float32)
    assert M.digit_exponent(4 * np.abs(gp[4]).max(axis=(1, 2))).max() == 27
    gt, at = torch.from_numpy(gp), torch.from_numpy(want_a)
    for dt, ndt in ((torch.float32, np.float32), (torch.float64, np.float64)):
        assert np.array_equal(M.fold_t(gt, at, H, H, dt).numpy(), M.fold(gp, want_a, H, H, ndt))
    want = torch.from_numpy(M.wgrad(frames, gp, want_a))
    got = M.wgrad_t(ft, None, gt, at, chunk=3)
    assert M.ulps(got.view(16, 36), want.float()).max().item() <= 1
    assert (got.double().view(16, 36) - want).abs().max().item() <= 2 ** -24 * want.abs().max().item()
    base = torch.from_numpy(rng.standard_normal((16, 4, 3, 3)).astype(np.float32))
    acc = M.wgrad_t(ft, None, gt, at, base=base)
    assert M.ulps(acc.view(16, 36), (base.double().view(16, 36) + want).float()).max().item() <= 1
