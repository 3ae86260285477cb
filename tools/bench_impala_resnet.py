"""Measure IMPALA, or R2D2, on the residual network (impala.resnet_small_model, r2d2.resnet_model) on one GPU.

    python tools/bench_impala_resnet.py [--steps 20] [--iters 20]
    python tools/bench_impala_resnet.py --workload r2d2 [--steps 20] [--iters 20]

--workload r2d2 prints, at B = 64, T = 80, MEM = 20 (1 280 burn-in and 3 840 window stacks per network):
  - the two-network stem launch (R.stem_fused_pair) against two single-net launches (R.stem_fused) on the same rows,
    at both stack counts, timed with CUDA events (burn-in: the pair without argmax; window: with the online argmax);
  - captured in-process learner steps/s and peak device memory for r2d2.resnet_model() and for the default conv model;
  - one eager residual-model step under torch.profiler: its kernels' device time split into stem, residual-block
    convs, LSTM, dense heads and the rest.

The default (IMPALA) workload:

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


def profile_step(L, classes=KERNEL_CLASSES) -> dict:
    """One eager step of learner L under torch.profiler: device time of its kernels by `classes`, and the largest
    six."""
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
        cls = next((c for c, keys in classes if any(k in name.lower() for k in keys)), "other")
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


# ---- --workload r2d2 ---------------------------------------------------------------------------------------------
R2D2_B, R2D2_T, R2D2_MEM, R2D2_N = 64, 80, 20, 160

LSTM = "LSTM (cuDNN RNN, cuBLAS GEMMs)"
R2D2_CLASSES = (                         # first match wins; names are the kernels' own
    ("stem", ("k_stem",)),
    ("dense heads (3xTF32, dueling tail)", ("k_gemm", "splitk", "dueling")),
    (LSTM, ("rnn", "lstm", "elemwise")),
    ("residual-block convs (cuDNN, with its layout transforms)",
     ("fprop", "dgrad", "wgrad", "implicit", "convolve", "winograd", "fft", "conv", "nchwtonhwc", "nhwctonchw")),
    (LSTM, ("gemm",)),                   # the only cuBLAS GEMMs left: the LSTM's input and recurrent projections
)


def r2d2_store(dev):
    """A stack store of R2D2_N hashed sequences, valid small fields and a built tree."""
    from distributed_rl_b200 import replay as R
    st = R.DeviceReplay(R2D2_N, R.r2d2_fields(R2D2_T), dev)
    fill_r2d2(st, 1)
    return st


def fill_r2d2(st, seed):
    st.fill_hash(R2D2_N, seed=seed)
    g = torch.Generator(device=st.device).manual_seed(seed)
    st.field_view("action").random_(0, 6, generator=g)
    st.field_view("reward").normal_(generator=g)
    for name in ("h0", "h1"):
        st.field_view(name).normal_(0.0, 0.1, generator=g)
    st.field_view("notdone").bernoulli_(0.9, generator=g)
    st.build(torch.rand(R2D2_N, generator=torch.Generator().manual_seed(seed)).to(st.device) + 0.05)


def r2d2_stem_pair(iters: int) -> dict:
    """The pair launch against two single-net launches over the rows of one B = 64 draw, burn-in and window."""
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.learner_common import time_major_rows
    dev = torch.device("cuda:0")
    st = r2d2_store(dev)
    frames = st.field_view("state").view(-1, 4, 84, 84)
    seq = torch.randperm(R2D2_N, device=dev)[:R2D2_B]
    rows = time_major_rows(seq, torch.arange(R2D2_T, device=dev).view(R2D2_T, 1))
    split = R2D2_MEM * R2D2_B
    on, tg = R.stem_pack_pair(dev)
    on.pack(torch.randn(16, 4, 3, 3, device=dev) * 0.1)
    tg.pack(torch.randn(16, 4, 3, 3, device=dev) * 0.1)
    out = {}
    for name, r, amax in (("burn_in", rows[:split], False), ("window", rows[split:], True)):
        n = r.numel()
        single = [(torch.empty(n, 16, 42, 42, device=dev), torch.empty(n, 16, 42, 42, dtype=torch.uint8, device=dev))
                  for _ in range(2)]
        pair = (torch.empty(2, n, 16, 42, 42, device=dev),
                torch.empty(n, 16, 42, 42, dtype=torch.uint8, device=dev) if amax else None)

        def two_singles():
            R.stem_fused(frames, r, on, out=single[0])
            R.stem_fused(frames, r, tg, out=single[1])

        def one_pair():
            R.stem_fused_pair(frames, r, on, tg, argmax=amax, out=pair)

        ms = {"two_singles": [], "pair": []}
        for _ in range(3):                                   # alternated, so that both see the same clocks
            ms["two_singles"].append(time_events(two_singles, iters))
            ms["pair"].append(time_events(one_pair, iters))
        torch.cuda.synchronize()
        for k in range(2):
            assert torch.equal(pair[0][k], single[k][0]), (name, k)
        if amax:
            assert torch.equal(pair[1], single[0][1]), name
        out[name] = {"stacks": n, "argmax": amax, "two_singles_ms": ms["two_singles"], "pair_ms": ms["pair"]}
    st.close()
    return out


def r2d2_steps(model: str, steps: int, profiled: bool) -> dict:
    from distributed_rl_b200 import r2d2
    dev = torch.device("cuda:0")
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    torch.manual_seed(0)
    cfg = r2d2.R2D2Config(BATCHSIZE=R2D2_B, FIXED_TRAJECTORY=R2D2_T, MEM=R2D2_MEM, REPLAY_MEMORY_LEN=R2D2_N,
                          LEARNER_DEVICE="cuda:0",
                          MODEL=r2d2.resnet_model() if model == "resnet" else r2d2.default_r2d2_model())
    L = r2d2.Learner(cfg, start_replay=False)
    fill_r2d2(L.memory.store, 1)
    L.fused_step(use_graph=True)                         # 3 eager warm-ups + capture
    for _ in range(3):
        L.fused_step(use_graph=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        L.fused_step(use_graph=True)
    torch.cuda.synchronize()
    out = {"steps_per_s": steps / (time.perf_counter() - t0),
           "peak_GB": torch.cuda.max_memory_allocated(dev) / 1e9,
           "params": sum(p.numel() for p in L.model.parameters())}
    if profiled:
        L._graph = None                                  # eager steps from here on
        out["eager_step_kernels"] = profile_step(L, R2D2_CLASSES)
    L.memory.store.close()
    del L
    torch.cuda.empty_cache()
    return out


def main_r2d2(args, info):
    res = dict(info, workload="r2d2", B=R2D2_B, T=R2D2_T, MEM=R2D2_MEM)
    pair = r2d2_stem_pair(args.iters)
    res["stem_pair"] = pair
    for name, p in pair.items():
        print(f"stem {name} ({p['stacks']} stacks per net, argmax {p['argmax']}): pair "
              f"{min(p['pair_ms']):.3f}-{max(p['pair_ms']):.3f} ms, two single-net launches "
              f"{min(p['two_singles_ms']):.3f}-{max(p['two_singles_ms']):.3f} ms")
    for rep in range(2):                                 # alternated, twice: the spread of the step rates
        for model in ("resnet", "conv"):
            s = r2d2_steps(model, args.steps, profiled=model == "resnet" and rep == 1)
            res.setdefault(f"{model}", []).append(s)
            print(f"r2d2 {model} ({s['params']} parameters) captured step B={R2D2_B} T={R2D2_T}: "
                  f"{s['steps_per_s']:.2f} steps/s, peak {s['peak_GB']:.2f} GB")
            split = s.get("eager_step_kernels")
            if split is not None:
                parts = ", ".join(f"{k} {v:.1f} ms" for k, v in split.items() if k not in ("total_ms", "top"))
                print(f"eager {model} step under torch.profiler: kernels {split['total_ms']:.1f} ms: {parts}")
                for ms, name in split["top"]:
                    print(f"    {ms:8.2f} ms  {name}")
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("impala", "r2d2"), default="impala")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_impala_resnet needs a CUDA device")
    info = card()
    print(f"# {info['gpu']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}")
    if args.workload == "r2d2":
        return main_r2d2(args, info)
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
