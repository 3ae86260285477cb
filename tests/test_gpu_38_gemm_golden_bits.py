"""The heads' 3xTF32 GEMM (csrc/gemm.cu) against recorded bits.

tests/golden/gemm_tf32x3_sm90.json holds, for every GEMM shape the Ape-X, R2D2 and IMPALA learners launch at
bench.py's configurations (plus a contraction length that is not a multiple of the 32-float chunk), the SHA-256 of
what the learner consumes: the K-split partials (b2rl_gemm_tf32x3_partials) or the reduced output
(b2rl_gemm_tf32x3).  The inputs are regenerated from the recorded recipe.  A change to how the operands are staged
must leave these bits alone; a changed bit in a priority changes every later sample.  The split count, and so the
bits, depend on the SM count: on a card with another count the test skips."""
import hashlib
import json
import os

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_tf32x3_sm90.json")


def inputs(entry):
    """A [M][K] and B [N][K], standard normal from a CPU generator seeded with entry["seed"] (A first)."""
    g = torch.Generator().manual_seed(entry["seed"])
    a = torch.randn(entry["M"], entry["K"], generator=g)
    b = torch.randn(entry["N"], entry["K"], generator=g)
    return a.cuda(), b.cuda()


def digest(entry):
    """-> (sha256 hex, splits) of the recorded call on this device."""
    from distributed_rl_b200 import linear as L
    M, N, K = entry["M"], entry["N"], entry["K"]
    a, b = inputs(entry)
    pa, pb = L.split_pack(a, False, False), L.split_pack(b, False, True)
    if entry["call"] == "partials":
        part, splits, ldc = L.gemm_partials(pa, pb, M, N, K)
        out = part.view(splits, M, ldc)[:, :, :N]
    else:
        out, splits = L.gemm_packed(pa, pb, M, N, K), None
        out = out[:, :N]
    torch.cuda.synchronize()
    return hashlib.sha256(out.contiguous().cpu().numpy().tobytes()).hexdigest(), splits


def _entries():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("entry", _entries()["shapes"], ids=lambda e: e["name"])
def test_gemm_bits_match_the_recording(entry):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    rec = _entries()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != rec["sms"]:
        pytest.skip(f"recorded on {rec['sms']} SMs, this device has {sms}: the K splits differ")
    got, splits = digest(entry)
    if entry["call"] == "partials":
        assert splits == entry["splits"], (splits, entry["splits"])
    assert got == entry["sha256"], f"{entry['name']}: {entry['M']} x {entry['N']} x {entry['K']} changed bits"
