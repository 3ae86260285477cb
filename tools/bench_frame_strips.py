"""R2D2 frame strips (R2D2Config.FRAME_STRIP) against frame stacks, measured in one command with alternating layouts.

    python tools/bench_frame_strips.py [--batch 64] [--steps 50] [--rounds 3] [--out DIR]

Prints one JSON line per measurement and a summary, with the card's name and power limit:
  * in-process: steps/s of the captured fused_step over a PAYLOAD_POOL store (2^14 distinct sequences behind 2^20
    tree slots), stacks and strips alternating;
  * served: steps/s of the captured bound step on the slots of a serve ring created in this process (ServeRing over
    a 2048-sequence store, filled once; each step binds the next slot as DeviceReplayClient.acquire does), alternating;
  * bytes per stored sequence, and free device memory before and after creating a 10^5-sequence strip store;
  * push_arrays sequences/s from pinned host buffers (strips handed over as strips, stacks as stacks).
Needs a GPU; there is no CPU fallback."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from distributed_rl_b200 import r2d2, replay as R  # noqa: E402
from distributed_rl_b200.replay_server import ServeRing  # noqa: E402

T = 80


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"card": q.stdout.strip() or torch.cuda.get_device_name(0)}


def _fill(store, n, seed):
    store.fill_hash(n, seed=seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    store.field_view("action").random_(0, 6, generator=g)
    store.field_view("reward").normal_(generator=g)
    for name in ("h0", "h1"):
        store.field_view(name).normal_(0.0, 0.1, generator=g)
    store.field_view("notdone").bernoulli_(0.9, generator=g)


def _timed(step, steps) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def in_process(strip: bool, B: int, steps: int, warmup: int) -> float:
    torch.manual_seed(0)
    cfg = r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=1 << 20, PAYLOAD_POOL=1 << 14,
                          FRAME_STRIP=strip, LEARNER_DEVICE="cuda:0")
    L = r2d2.Learner(cfg, start_replay=False)
    _fill(L.memory.pool, 1 << 14, 5)
    L.memory.store.build(torch.rand(1 << 20, device="cuda") + 0.05)
    L.memory.store.seed(1, 0)
    for _ in range(warmup):
        L.fused_step(use_graph=True)
    rate = _timed(lambda: L.fused_step(use_graph=True), steps)
    L.memory.store.close(), L.memory.pool.close()
    del L
    torch.cuda.empty_cache()
    return rate


def served(strip: bool, B: int, steps: int, warmup: int) -> float:
    slots = steps + warmup + 4
    fields = R.r2d2_fields(T, strip=strip)
    n = 2048
    st = R.DeviceReplay(n, fields, "cuda:0")
    _fill(st, n, 7)
    st.build(torch.rand(n, device="cuda") + 0.05)
    st.seed(3, 0)
    slot_rows = min(slots, 16)
    ring = ServeRing.create(st, B, slot_rows)
    for k in range(slot_rows):
        ring.fill(st, k, k + 1, 0.4)
    torch.manual_seed(0)
    mem = SimpleNamespace(ring=ring, acquire=None, release=None, is_alive=lambda: True)
    L = r2d2.Learner(r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=8, FRAME_STRIP=strip,
                                     SERVED_FUSED_STEP=True, LEARNER_DEVICE="cuda:0"), start_replay=False, memory=mem)
    s = L._state()
    k = [0]

    def step():
        ring.bind(ring.slot_ptrs(k[0] % slot_rows)[0][0], fields, s.cur, s.frames, torch.cuda.current_stream())
        L._bound_step()
        k[0] += 1
    for _ in range(warmup):
        step()
    rate = _timed(step, steps)
    ring.close()
    st.close()
    del L
    torch.cuda.empty_cache()
    return rate


def capacity() -> dict:
    per = {name: sum(f.nbytes for f in R.r2d2_fields(T, strip=s)) for name, s in (("stacks", False), ("strips", True))}
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    st = R.DeviceReplay(100_000, R.r2d2_fields(T, strip=True), "cuda:0")
    st.fill_hash(100_000, seed=1)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    st.close()
    torch.cuda.synchronize()
    return {"bytes_per_sequence": per, "total_bytes": total, "free_before_100k_strip_store": free0,
            "free_after_100k_strip_store": free1, "store_bytes_measured": free0 - free1}


def push_rate(strip: bool, n: int, reps: int) -> float:
    cfg = r2d2.R2D2Config(BATCHSIZE=32, FIXED_TRAJECTORY=T, REPLAY_MEMORY_LEN=4 * n, FRAME_STRIP=strip,
                          LEARNER_DEVICE="cuda:0")
    rp = r2d2.Replay(cfg)
    shape = (n, T + 3, 84, 84) if strip else (n, T, 4, 84, 84)
    cols = [torch.randint(0, 256, shape, dtype=torch.uint8).pin_memory(),
            torch.zeros(n, T, dtype=torch.int32).pin_memory(), torch.zeros(n, T).pin_memory(),
            torch.zeros(n, 512).pin_memory(), torch.zeros(n, 512).pin_memory(), torch.ones(n).pin_memory(),
            torch.ones(n).pin_memory()]
    rp.push_arrays(*cols)
    rate = _timed(lambda: rp.push_arrays(*cols), reps) * n
    rp.store.close()
    return rate


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--push-n", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res = dict(_card(), batch=a.batch, steps=a.steps, rounds=a.rounds, in_process={"stacks": [], "strips": []},
               served={"stacks": [], "strips": []}, push_seq_per_s={"stacks": [], "strips": []})
    for r in range(a.rounds):
        for name, strip in (("stacks", False), ("strips", True)) if r % 2 == 0 else (("strips", True), ("stacks", False)):
            res["in_process"][name].append(in_process(strip, a.batch, a.steps, a.warmup))
            res["served"][name].append(served(strip, a.batch, a.steps, a.warmup))
            res["push_seq_per_s"][name].append(push_rate(strip, a.push_n, 10))
            print(json.dumps({"round": r, "layout": name, "in_process": res["in_process"][name][-1],
                              "served": res["served"][name][-1], "push": res["push_seq_per_s"][name][-1]}), flush=True)
    res["capacity"] = capacity()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_frame_strips.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
