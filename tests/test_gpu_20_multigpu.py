"""Multi-GPU parity (SURVEY.md §8e) on real GPUs over NCCL: needs >= 2 GPUs, skipped otherwise.
The checks themselves live in tests/mgpu_worker.py (one process per GPU under torchrun)."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _run_worker(extra_env=None):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), os.path.join(HERE, "mgpu_worker.py")]
    env = dict(os.environ, **(extra_env or {}))
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("MGPU_OK") == 2, r.stdout[-3000:]
    return r.stdout


def test_data_parallel_gradient_equals_concatenated_batch_gradient():
    """Default configuration: heads over NCCL (overlapped), the late slice through libb2rl's peer-memory kernel."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    out = _run_worker()
    assert "peer_allreduce True" in out, out[-2000:]


@pytest.mark.parametrize("env", [{"B2RL_PEER_ALLREDUCE_BIG": "1"}, {"B2RL_NO_PEER_ALLREDUCE": "1"}],
                         ids=["heads_over_peer_memory", "nccl_only"])
def test_data_parallel_other_collective_paths(env):
    """The same parity checks with the heads' reduce-scatter + all-gather kernel switched on (opt-in) and with
    every collective on NCCL (what a multi-node run uses)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    out = _run_worker(env)
    if "B2RL_PEER_ALLREDUCE_BIG" in env:
        assert "heads True" in out, out[-2000:]
    else:
        assert "peer_allreduce False" in out, out[-2000:]
