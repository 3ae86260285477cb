"""The deduplicated Ape-X store with its frames stored encoded (ApexConfig.FRAME_CODEC), measured in one command.

    python tools/bench_apex_pool_codec.py [--batch 512] [--steps 100] [--rounds 3] [--slots 65536]

Every frame here is SYNTHETIC: tests/pool_codec_model.py renders Atari-like frames and tests/apex_atari_records.py
pairs their stacks as the reference Ape-X actors do (32 interleaved actors, s' UNROLL_STEP = 3 steps later).  There is
no emulator on the machines this runs on, so no ratio below is a ratio on real Atari frames.  The stores are filled
by pushing one block of such records from pinned buffers, over and over (so later copies are mostly dedup hits).
Prints, with the card's name, power limit and maximum SM clock:
  * bytes per stored frame: b2rl_frame_encode on the block's distinct frames and on uniformly random frames, and the
    coded store's codec_stats() after it is filled;
  * push: push_arrays records/s from pinned buffers while a raw FRAME_DEDUP store ("raw") and a FRAME_CODEC store
    ("coded") are filled;
  * step: steps/s of the captured fused_step at B = --batch, raw against coded, alternating, --rounds rounds each;
  * kernels: ms by CUDA events of conv_1's forward of s (one network), of s' (two networks) and of its weight
    gradient, on the raw pool ("raw"), on the coded pool decoded in conv_1's loader ("in-loader"), and as the gather
    that decodes s and s' into staged stacks plus conv_1 on them ("staged");
  * capacity: a 2^21-transition coded store created at DEDUP_WINDOW 2^20 and 2^16, its ring sized from the bytes per
    frame and new frames per record measured above: device bytes (torch.cuda.mem_get_info).
Needs a GPU; there is no CPU fallback."""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributed_rl_b200 import apex, replay as R  # noqa: E402
from apex_atari_records import atari_records  # noqa: E402

KINDS = ("raw", "coded")


def _card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _block(n, push_batch):
    recs = atari_records(n, actors=32, episode=400, seed=1)
    p = (np.random.default_rng(2).random(n) + 0.05).astype(np.float32)
    out = []
    for i in range(0, n, push_batch):
        chunk = []
        for x in (*recs, p):
            t = torch.from_numpy(np.ascontiguousarray(x[i:i + push_batch]))
            pin = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
            pin.copy_(t)
            chunk.append(pin)
        out.append(chunk)
    return out, recs


def _fill(memory, block, n) -> float:
    torch.cuda.synchronize()
    t0, done = time.perf_counter(), 0
    while done < n:
        for chunk in block:
            if done >= n:
                break
            memory.push_arrays(*chunk)
            done += chunk[-1].numel()
    torch.cuda.synchronize()
    return done / (time.perf_counter() - t0)


def _events(fn, n) -> float:
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--slots", type=int, default=65536)
    ap.add_argument("--block", type=int, default=16384)
    ap.add_argument("--kernel-iters", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": _card(), "batch": a.batch, "slots": a.slots, "frames": "synthetic Atari-like"}
    block, recs = _block(a.block, 512)

    # bytes per frame
    distinct = np.unique(np.concatenate([recs[0][:2048], recs[1][:2048]], axis=1).reshape(-1, 84 * 84), axis=0)
    _, units = R.encode_frames(torch.from_numpy(distinct).cuda().view(-1, 84, 84))
    rnd = torch.randint(0, 256, (1024, 84, 84), dtype=torch.uint8, device="cuda")
    _, ru = R.encode_frames(rnd)
    res["bytes_per_frame_synthetic"] = 16.0 * units.double().mean().item()
    res["bytes_per_frame_random"] = 16.0 * ru.double().mean().item()

    # stores, filled alternately: push rate
    learners, push = {}, {k: [] for k in KINDS}
    for kind in KINDS:
        cfg = apex.ApexConfig(BATCHSIZE=a.batch, REPLAY_MEMORY_LEN=a.slots, BUFFER_SIZE=0, LEARNER_DEVICE="cuda:0",
                              FRAME_DEDUP=True, FRAME_CODEC=kind == "coded")
        torch.manual_seed(0)
        learners[kind] = apex.Learner(cfg, connect=None, start_replay=False)
    for r in range(a.rounds):
        for kind in KINDS:
            push[kind].append(_fill(learners[kind].memory, block, a.slots if r == 0 else a.block))
    coded_store = learners["coded"].memory.store
    cs = coded_store.codec_stats()
    res["codec_stats"] = cs
    # the block's distinct frames per record: later copies of the block are (mostly) dedup hits
    res["new_frames_per_record"] = cs["frames_stored"] / min(a.slots, a.block)
    res["push_records_per_s"] = push

    # captured step, alternating
    steps = {k: [] for k in KINDS}
    for kind in KINDS:
        learners[kind].memory.store.seed(5, 0)
        for _ in range(10):
            learners[kind].fused_step(use_graph=True)
    for _ in range(a.rounds):
        for kind in KINDS:
            L = learners[kind]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                L.fused_step(use_graph=True)
            torch.cuda.synchronize()
            steps[kind].append(a.steps / (time.perf_counter() - t0))
    res["captured_step_per_s"] = steps

    # conv_1 kernels: raw pool, coded in-loader, gather-decode + conv_1 on staged stacks
    raw_store = learners["raw"].memory.store
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    idx = torch.randint(0, a.slots, (a.batch,), device="cuda", generator=g)
    p1, p2 = R.Conv1Pack(1, "cuda"), R.Conv1Pack(2, "cuda")
    w = torch.randn(32, 4, 8, 8, device="cuda", generator=g) * 0.05
    for p in (p1, p2):
        for k in range(p.n_nets):
            p.pack(k, w)
    gy = torch.randn(a.batch, 32, 20, 20, device="cuda", generator=g)
    out1 = torch.empty(1, a.batch, 20, 20, 32, device="cuda")
    out2 = torch.empty(2, a.batch, 20, 20, 32, device="cuda")
    gw = torch.empty(32, 4, 8, 8, device="cuda")
    staged = coded_store.alloc_batch(a.batch, ("state", "next_state"))

    def arms():
        for name, st in (("raw", raw_store), ("in-loader", coded_store)):
            s, ns = st.frame_source("state"), st.frame_source("next_state")
            yield name, (lambda i, s=s: R.conv1_fused(s, idx, p1, relu=True, out=out1),
                         lambda i, ns=ns: R.conv1_fused(ns, idx, p2, relu=False, out=out2),
                         lambda i, s=s: R.conv1_wgrad(s, idx, gy, out=gw))
        yield "staged", (lambda i: (coded_store.gather(idx, {"state": staged["state"], "next_state": None}),
                                    R.conv1_fused(staged["state"], None, p1, relu=True, out=out1)),
                         lambda i: (coded_store.gather(idx, {"next_state": staged["next_state"], "state": None}),
                                    R.conv1_fused(staged["next_state"], None, p2, relu=False, out=out2)),
                         lambda i: R.conv1_wgrad(staged["state"], None, gy, out=gw))

    kern = {}
    for name, fns in arms():
        for fn in fns:
            _events(fn, 5)
    for _ in range(a.rounds):
        for name, fns in arms():
            kern.setdefault(name, []).append([round(_events(fn, a.kernel_iters), 4) for fn in fns])
    res["kernel_ms_fwd_s_fwd_ns_wgrad"] = kern
    y_in = R.conv1_fused(coded_store.frame_source("next_state"), idx, p2)
    coded_store.gather(idx, {"next_state": staged["next_state"], "state": None})
    y_st = R.conv1_fused(staged["next_state"], None, p2)
    res["in_loader_equals_staged"] = all(torch.equal(u, v) for u, v in zip(y_in, y_st))
    del learners, raw_store, coded_store, staged
    gc.collect()
    torch.cuda.empty_cache()

    # capacity of a 2^21-transition coded store
    n = 1 << 21
    per_record = res["new_frames_per_record"] * res["bytes_per_frame_synthetic"]
    cap = {}
    for W in (1 << 20, 1 << 16):
        cfg = apex.ApexConfig(REPLAY_MEMORY_LEN=n, FRAME_DEDUP=True, FRAME_CODEC=True, DEDUP_WINDOW=W,
                              POOL_BYTES_PER_TRANSITION=(7072 * (W + 10) + 1.25 * per_record * n) / n)
        F, W_ = apex.dedup_geometry(cfg)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        st = R.CodedDedupReplay(n, F, W_, apex.pool_bytes(cfg))
        torch.cuda.synchronize()
        cap[f"W=2^{W.bit_length() - 1}"] = {"pool_bytes": apex.pool_bytes(cfg),
                                            "device_bytes": free0 - torch.cuda.mem_get_info()[0]}
        del st
        gc.collect()
        torch.cuda.empty_cache()
    res["capacity_2^21"] = cap
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
