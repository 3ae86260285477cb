"""Time the heads' 3xTF32 GEMM (csrc/gemm.cu) at the shapes the learner steps run, as the step runs them.

Each call is captured 20 times back to back in a CUDA graph with its operands L2-warm, like bench.py's captured step;
the best of 15 replays is reported.  Calls the learner makes through b2rl_gemm_tf32x3_partials are timed as
k_gemm_tf32x3 alone, the others with their k_splitk_reduce.  Per shape it prints:
  * the time and the floor at the data sheet's dense TF32 rate (495 TFLOP/s on an H100 SXM at 700 W: 3 TF32
    products per fp32 multiply-add),
  * achieved TF32 TFLOP/s (6 M N K / time),
  * the rate at which the CTAs stage operand tiles from L2 / HBM into shared memory: every CTA loads the {hi, lo}
    tiles of both operands, (128 + 256) rows x 8 B per contraction element over its K range.

    python tools/bench_gemm.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from distributed_rl_b200 import linear as L

TF32_PEAK = 495e12
TM, TN, KC = 128, 256, 32          # gemm.cu's tiles and contraction padding

# (learner, call, M, N, K, "partials" | "output"): every GEMM the learners launch at bench.py's configurations
# (tests/golden/gemm_tf32x3_sm90.json records the same list)
SHAPES = [
    ("apex", "online forward (s ++ s')", 1024, 1024, 3136, "partials"),
    ("apex", "target forward", 512, 1024, 3136, "partials"),
    ("apex", "dL/dx", 512, 3136, 1024, "partials"),
    ("apex", "dL/dW", 1024, 3136, 512, "output"),
    ("r2d2", "forward", 1280, 1024, 512, "output"),
    ("r2d2", "forward", 3840, 1024, 512, "output"),
    ("r2d2", "dL/dW", 1024, 512, 3840, "output"),
    ("r2d2", "dL/dx", 3840, 512, 1024, "output"),
    ("impala", "forward", 1024, 256, 2592, "output"),
    ("impala", "forward", 20480, 256, 2592, "output"),
    ("impala", "dL/dW", 256, 2592, 20480, "output"),
    ("impala", "dL/dx", 20480, 2592, 256, "output"),
]


def warm(fn, reps=20, rounds=15):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3 / reps)
    return best


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py needs a CUDA device")
    p = torch.cuda.get_device_properties(0)
    print(f"{p.name}, {p.multi_processor_count} SMs")
    print(f"{'learner':7s} {'call':26s} {'M x N x K':>20s} {'us':>7s} {'floor':>6s} {'TFLOP/s':>8s} {'stage TB/s':>10s}")
    for learner, call, M, N, K, kind in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        a = L.split_pack(torch.randn(M, K, device="cuda", generator=g), False, False)
        b = L.split_pack(torch.randn(N, K, device="cuda", generator=g), False, True)
        if kind == "partials":
            fn = lambda: L.gemm_partials(a, b, M, N, K)
        else:
            out = torch.empty(M, (N + 3) // 4 * 4, device="cuda")[:, :N]
            fn = lambda: L.gemm_packed(a, b, M, N, K, out=out)
        us = warm(fn)
        flop = 6.0 * M * N * K
        k_pad = (K + KC - 1) // KC * KC
        staged = -(-M // TM) * -(-N // TN) * (TM + TN) * 8 * k_pad
        print(f"{learner:7s} {call:26s} {f'{M} x {N} x {K}':>20s} {us:7.1f} {flop / TF32_PEAK * 1e6:6.1f} "
              f"{flop / us / 1e6:8.0f} {staged / us / 1e6:10.2f}")


if __name__ == "__main__":
    main()
