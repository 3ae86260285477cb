"""CPU tests of R2D2 on the IMPALA residual network (r2d2.resnet_model()): the model's layers and parameter count, the
round trip through the drop-in `configuration` module, the reference actor's side (the drop-in baseAgent loading the
learner's weights and carrying its LSTM state across single-frame calls), and the refusals that need no GPU."""
import json
import os
import subprocess
import sys
import textwrap
import types

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def test_the_model_is_the_default_net_with_the_residual_torso():
    from distributed_rl_b200 import impala, r2d2
    from distributed_rl_b200.agent import GraphAgent, ResidualStack
    m = r2d2.resnet_model()
    d = r2d2.default_r2d2_model()
    assert m["module00"] == impala.resnet_small_model()["module00"] and m["module02"]["iSize"] == 3872
    assert {k: v for k, v in m.items() if k not in ("module00", "module02")} == \
        {k: v for k, v in d.items() if k not in ("module00", "module02")}
    assert {k: v for k, v in m["module02"].items() if k != "iSize"} == \
        {k: v for k, v in d["module02"].items() if k != "iSize"}
    assert r2d2.resnet_model() == m and d == r2d2.default_r2d2_model()       # fresh dicts, the default untouched
    net = GraphAgent(m)
    assert isinstance(net.module00, ResidualStack) and net.first_stem_node() == "module00"
    assert net.first_conv_node() is None
    count = {n: sum(p.numel() for p in getattr(net, n).parameters()) for n in ("module00", "module02")}
    assert count == {"module00": 97_344, "module02": 8_982_528}
    assert sum(p.numel() for p in net.parameters()) == 9_607_744
    assert sum(p.numel() for p in GraphAgent(d).parameters()) == 8_080_896
    keys = set(net.state_dict())
    want = {"module00.conv_1.weight", "module00.block_1_1.conv_1.weight", "module00.block_3_2.conv_2.weight",
            "module02.rnn.weight_ih_l0", "module02.rnn.weight_hh_l0", "module03.MLP_1.weight", "module03.MLP_2.weight",
            "module03_1.MLP_1.weight", "module03_1.MLP_2.weight"}
    assert want <= keys
    assert net.state_dict()["module02.rnn.weight_ih_l0"].shape == (4 * 512, 3872)
    assert {k for k in keys if not k.startswith("module00.")} == \
        {k for k in GraphAgent(d).state_dict() if not k.startswith("module00.")}


def test_the_forward_from_the_stem_is_the_forward():
    """forward_from_stem(pool_1(conv_1(x)), [shape]) is forward([x, shape]): what the fused learner runs."""
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200.agent import GraphAgent
    torch.manual_seed(0)
    net = GraphAgent(r2d2.resnet_model())
    T, B = 3, 2
    x = torch.rand(T * B, 4, 84, 84)
    shape = torch.tensor([T, B, -1])
    hc = (torch.randn(1, B, 512) * 0.1, torch.randn(1, B, 512) * 0.1)
    net.setCellState(hc)
    want = net.forward([x, shape])[0]
    net.setCellState(hc)
    got = net.forward_from_stem(net.module00.pool_1(net.module00.conv_1(x)), [shape])[0]
    assert want.shape == (T * B, 6)
    torch.testing.assert_close(got, want, rtol=0, atol=0)


def _run(code, tmp_path, cfg):
    (tmp_path / "cfg").mkdir(exist_ok=True)
    (tmp_path / "cfg" / "r2d2.json").write_text(json.dumps(cfg))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(REPO, "dropin"), REPO]),
               B2RL_CFG=str(tmp_path / "cfg" / "r2d2.json"))
    return subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=tmp_path, env=env, capture_output=True,
                          text=True, timeout=300)


def _r2d2_json():
    from distributed_rl_b200 import r2d2
    d = r2d2.R2D2Config()
    return {"ALG": "R2D2", "REDIS_SERVER": "localhost", "ACTION_SIZE": d.ACTION_SIZE, "ALPHA": d.ALPHA,
            "BETA": d.BETA, "GAMMA": d.GAMMA, "TARGET_FREQUENCY": d.TARGET_FREQUENCY, "N": 8,
            "BATCHSIZE": d.BATCHSIZE, "DEVICE": "cpu", "LEARNER_DEVICE": "cpu",
            "REPLAY_MEMORY_LEN": d.REPLAY_MEMORY_LEN, "BUFFER_SIZE": d.BUFFER_SIZE, "UNROLL_STEP": d.UNROLL_STEP,
            "FIXED_TRAJECTORY": d.FIXED_TRAJECTORY, "MEM": d.MEM, "USE_RESCALING": d.USE_RESCALING,
            "optim": d.OPTIM_INFO, "model": r2d2.resnet_model()}


def test_the_config_round_trip_and_the_actor_side(tmp_path):
    """cfg/r2d2.json with the residual model -> configuration -> R2D2Config.from_configuration(); then the actor's
    side: the drop-in baseAgent built from the same MODEL loads the learner's state_dict and steps one frame at a time
    with a [1, 1, -1] shape, carrying (h, c) from one call to the next."""
    r = _run("""
        import torch
        import configuration as C
        from distributed_rl_b200 import r2d2
        from distributed_rl_b200.agent import GraphAgent
        from baseline.baseAgent import baseAgent
        cfg = r2d2.R2D2Config.from_configuration()
        assert cfg.MODEL == r2d2.resnet_model() and cfg.FUSED_CONV1
        assert cfg == r2d2.R2D2Config(MODEL=r2d2.resnet_model(), LEARNER_DEVICE="cpu", LOG_W=C.LOG_W)
        torch.manual_seed(0)
        learner = GraphAgent(cfg.MODEL)            # what Learner.state_dict publishes: the online net's weights
        sd = {k: v.cpu() for k, v in learner.state_dict().items()}
        torch.manual_seed(1)
        actor = baseAgent(C.MODEL)
        actor.load_state_dict(sd)
        for k, v in actor.state_dict().items():
            assert torch.equal(v, sd[k]), k
        shape = torch.tensor([1, 1, -1])
        actor.zeroCellState()
        frames = torch.rand(2, 1, 4, 84, 84)
        q0 = actor.forward([frames[0], shape])[0]
        h1 = actor.getCellState()
        q1 = actor.forward([frames[1], shape])[0]
        assert q0.shape == q1.shape == (1, C.ACTION_SIZE)
        assert h1[0].shape == (1, 1, 512) and bool(h1[0].abs().sum() > 0)
        # the second call started from the first call's (h, c): the same as one two-step call
        learner.zeroCellState()
        both = learner.forward([frames.view(2, 4, 84, 84), torch.tensor([2, 1, -1])])[0]
        torch.testing.assert_close(both, torch.cat([q0, q1]), rtol=1e-5, atol=1e-6)
        actor.zeroCellState()
        assert not torch.allclose(actor.forward([frames[1], shape])[0], q1)
        print("OK")
    """, tmp_path, _r2d2_json())
    assert r.returncode == 0, r.stderr
    assert "OK" in r.stdout


def _non_fused_resnet():
    """A RESCNN2D torso the stem kernels do not run: 32 channels in the first section."""
    from distributed_rl_b200 import r2d2
    from distributed_rl_b200.agent import GraphAgent
    m = r2d2.resnet_model()
    m["module00"]["nUnit"] = [32, 32, 32]
    net = GraphAgent(m)
    assert net.first_stem_node() is None and net.first_conv_node() is None
    return net


@pytest.mark.parametrize("served,what", [(True, "SERVED_FUSED_STEP"), (False, r"fused_step\(use_graph=True\)")])
def test_the_step_state_refuses_a_stem_the_kernels_do_not_run(served, what):
    from distributed_rl_b200 import r2d2
    L = types.SimpleNamespace(model=_non_fused_resnet(), cfg=r2d2.R2D2Config(), device=torch.device("cpu"),
                              _served=served)
    with pytest.raises(ValueError, match=what + ".*RESCNN2D stem"):
        r2d2._StepState(L)


def test_the_shared_predicate():
    from distributed_rl_b200 import apex, impala, r2d2
    from distributed_rl_b200.agent import GraphAgent
    from distributed_rl_b200.learner_common import fused_first_layer, require_fused_first_layer
    for m in (r2d2.resnet_model(), r2d2.default_r2d2_model(), impala.resnet_small_model(), apex.default_apex_model()):
        assert fused_first_layer(GraphAgent(m))
        require_fused_first_layer(GraphAgent(m), "x")
    assert not fused_first_layer(_non_fused_resnet())
    with pytest.raises(ValueError, match="the step.*RESCNN2D stem"):
        require_fused_first_layer(_non_fused_resnet(), "the step")
