"""Measure IMPALA on the residual network (impala.resnet_small_model) on one GPU.

    python tools/bench_impala_resnet.py [--steps 20] [--iters 20]

Prints, with the card's name and power limit read in the same run:
  - captured in-process learner steps/s at B = 32 and B = 1024 (T = 20), over a pushed stack store;
  - the fused stem (csrc/stem.cu) forward and weight gradient alone over one B = 1024 draw ((T + 1) B = 21 504 frame
    stacks), timed with CUDA events, against the unfused PyTorch stem on the same draw (gather, /255, cuDNN conv,
    max_pool2d, and their backward);
  - the stem's HBM bytes from the shapes and the achieved GB/s;
  - one eager B = 1024 step under torch.profiler (a run of its own, after the timed ones): its kernels' device time by
    class (stem, cuDNN convs, max-pool, dense heads, other) and the six largest kernels.
The last line is one JSON object with every number."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

T = 20
STACK = 4 * 84 * 84                  # uint8 bytes of one frame stack
POOLED = 16 * 42 * 42                # pooled elements per stack


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[0].split(",")] if q else (torch.cuda.get_device_name(), "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def rollouts(n: int, seed: int):
    """n rollouts of frames with flat regions and noise (Atari-like statistics are not needed for timing)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (n, T + 1, 4, 21, 21), dtype=torch.uint8, generator=g)
    state = base.repeat_interleave(4, dim=3).repeat_interleave(4, dim=4).reshape(n, T + 1, STACK).contiguous()
    a = torch.randint(0, 6, (n, T), dtype=torch.int32, generator=g)
    mu = torch.rand(n, T, generator=g) * 0.8 + 0.1
    r = torch.randn(n, T, generator=g)
    done = (torch.rand(n, generator=g) > 0.1).float()
    return [state, a, mu, r, done]


def time_events(fn, iters: int) -> float:
    """Mean milliseconds of fn() over `iters` calls, between CUDA events (after two warm-up calls)."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


KERNEL_CLASSES = (                       # first match wins; names are the kernels' own
    ("stem", ("k_stem",)),
    ("conv (cuDNN)", ("cudnn", "xmma", "implicit", "convolve", "fprop", "wgrad", "dgrad", "winograd", "fft")),
    ("max-pool", ("max_pool", "maxpool")),
    ("dense heads (3xTF32)", ("k_gemm", "splitk")),
)


def profile_step(L) -> dict:
    """One eager step of learner L under torch.profiler: device time of its kernels by class, and the largest six."""
    from torch.profiler import ProfilerActivity, profile
    L.fused_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        L.fused_step()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        per[e.name] = per.get(e.name, 0.0) + e.time_range.elapsed_us() / 1000.0
    split = {"total_ms": sum(per.values())}
    for name, ms in per.items():
        cls = next((c for c, keys in KERNEL_CLASSES if any(k in name.lower() for k in keys)), "other")
        split[cls] = split.get(cls, 0.0) + ms
    split["top"] = sorted(((ms, name[:90]) for name, ms in per.items()), reverse=True)[:6]
    return split


def learner_steps(B: int, steps: int, cols, profiled: bool = False):
    from distributed_rl_b200 import impala
    torch.manual_seed(0)
    N = cols[-1].numel()
    L = impala.Learner(impala.ImpalaConfig(BATCHSIZE=B, UNROLL_STEP=T, REPLAY_MEMORY_LEN=N, LEARNER_DEVICE="cuda:0",
                                           MODEL=impala.resnet_small_model()), start_replay=False)
    L.memory.push_arrays(*cols)
    L.fused_step(use_graph=True)                         # 3 eager warm-ups + capture
    for _ in range(3):
        L.fused_step(use_graph=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        L.fused_step(use_graph=True)
    torch.cuda.synchronize()
    sps = steps / (time.perf_counter() - t0)
    split = profile_step(L) if profiled else None
    del L
    torch.cuda.empty_cache()
    return sps, split


def stem_alone(iters: int, cols) -> dict:
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.learner_common import time_major_rows
    F = torch.nn.functional
    B, N = 1024, cols[-1].numel()
    dev = torch.device("cuda:0")
    st = R.DeviceReplay(N, R.impala_fields(T), dev)
    st.push(cols, torch.ones(N))
    frames = st.field_view("state").view(-1, 4, 84, 84)
    idx = torch.randperm(N, device=dev)[:B]
    rows = time_major_rows(idx, torch.arange(T + 1, device=dev).view(T + 1, 1))
    n = rows.numel()
    w = (torch.randn(16, 4, 3, 3, device=dev) * 0.1)
    pack = R.StemPack(dev)
    pack.pack(w)
    pooled, amax = R.stem_fused(frames, rows, pack)
    gp = torch.randn(n, 16, 42, 42, device=dev)
    out = {"rows": n}
    out["fused_fwd_ms"] = time_events(lambda: R.stem_fused(frames, rows, pack, out=(pooled, amax)), iters)
    gw = torch.empty(16, 4, 3, 3, device=dev)
    out["fused_wgrad_ms"] = time_events(lambda: R.stem_wgrad(frames, rows, gp, amax, out=gw), iters)
    wl = w.clone().requires_grad_(True)

    def unfused_fwd():
        x = frames.index_select(0, rows).float().div_(255.0)
        return F.max_pool2d(F.conv2d(x, wl, padding=1), 3, 2, 1)

    def unfused_fwd_bwd():
        wl.grad = None
        unfused_fwd().backward(gp)

    with torch.no_grad():
        out["unfused_fwd_ms"] = time_events(unfused_fwd, iters)
    out["unfused_fwd_bwd_ms"] = time_events(unfused_fwd_bwd, iters)
    out["unfused_bwd_ms"] = out["unfused_fwd_bwd_ms"] - out["unfused_fwd_ms"]
    # bytes the fused kernels must move: frames in, pooled fp32 + uint8 argmax out; backward the same three back in
    fwd_bytes = n * (STACK + POOLED * 4 + POOLED)
    out["fused_fwd_GB"] = fwd_bytes / 1e9
    out["fused_wgrad_GB"] = fwd_bytes / 1e9
    out["fused_fwd_GBps"] = fwd_bytes / out["fused_fwd_ms"] / 1e6
    out["fused_wgrad_GBps"] = fwd_bytes / out["fused_wgrad_ms"] / 1e6
    out["cudnn_allow_tf32"] = torch.backends.cudnn.allow_tf32
    st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_impala_resnet needs a CUDA device")
    info = card()
    print(f"# {info['gpu']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}")
    cols = rollouts(1100, 0)
    res = dict(info)
    s = stem_alone(args.iters, cols)
    res["stem"] = s
    print(f"stem B=1024 T=20 ({s['rows']} stacks): fused fwd {s['fused_fwd_ms']:.3f} ms "
          f"({s['fused_fwd_GBps']:.0f} GB/s of {s['fused_fwd_GB']:.2f} GB), fused wgrad {s['fused_wgrad_ms']:.3f} ms "
          f"({s['fused_wgrad_GBps']:.0f} GB/s); unfused PyTorch fwd {s['unfused_fwd_ms']:.3f} ms, "
          f"bwd {s['unfused_bwd_ms']:.3f} ms (cuDNN allow_tf32={s['cudnn_allow_tf32']})")
    for B in (32, 1024):
        sps, split = learner_steps(B, args.steps, cols, profiled=B == 1024)
        res[f"steps_per_s_B{B}"] = sps
        print(f"resnet_small captured step B={B} T=20: {sps:.2f} steps/s ({sps * B * T:.0f} frames/s)")
        if split is not None:
            res[f"eager_step_kernels_B{B}"] = split
            parts = ", ".join(f"{k} {v:.1f} ms" for k, v in split.items() if k not in ("total_ms", "top"))
            print(f"eager step B={B} under torch.profiler: kernels {split['total_ms']:.1f} ms: {parts}")
            for ms, name in split["top"]:
                print(f"    {ms:8.2f} ms  {name}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
