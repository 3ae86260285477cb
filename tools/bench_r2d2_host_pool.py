"""The deduplicated R2D2 store with its frame pool in pinned host memory (R2D2Config.HOST_POOL), measured in one command.

    python tools/bench_r2d2_host_pool.py [--batch 64] [--steps 100] [--rounds 3] [--seqs 16384] [--max-host-gb 200]

Sequences are generated on the host as the reference R2D2 actors send them (tests/strip_dedup_model.py, 32 interleaved
actors); the stores are filled by pushing one block of 2048 such sequences from pinned buffers, over and over (a copy
older than the dedup window is stored again, so the stores hold every frame each time).  Prints, with the card's name,
power limit and maximum SM clock:
  * in-process: steps/s of the captured fused_step at B = --batch over --seqs sequences, on an HBM-pool dedup store
    ("hbm_pool"), a host-pool dedup store ("host_pool") and a HOST_FRAMES strip store ("host_frames"), the three
    alternating, --rounds rounds each;
  * push: push_arrays sequences/s from pinned buffers while those stores are filled;
  * gather: GB/s of the host-plane gather (k_gather_host_planes: B strips of scattered pool frames) against the
    host-row gather (k_gather_host_rows: B contiguous strips), the same minibatch bytes;
  * serve fill: ms of one b2rl_serve_fill from each dedup store;
  * capacity: the largest host-pool store of 2^K sequences (K >= 17) the host limit allows, filled past its slot ring's
    wrap: device bytes (torch.cuda.mem_get_info) and pinned bytes.
Host memory is shared: no store pins more than --max-host-gb or half of MemAvailable; a store that would is not created
and is reported as not measured.  Needs a GPU; there is no CPU fallback."""
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

from distributed_rl_b200 import r2d2, replay as R  # noqa: E402
from distributed_rl_b200.replay_server import ServeRing  # noqa: E402
from strip_dedup_model import player_sequences  # noqa: E402

T = 80
BLOCK = 2048
STRIP_BYTES = (T + 3) * R.FRAME_BYTES
KINDS = ("hbm_pool", "host_pool", "host_frames")


def _card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def host_limit(max_host_gb: float) -> int:
    with open("/proc/meminfo") as f:
        avail = next(int(line.split()[1]) * 1024 for line in f if line.startswith("MemAvailable"))
    return int(min(max_host_gb * 1e9, avail / 2))


def _cfg(kind, slots, batch, **kw):
    dedup = kind != "host_frames"
    return r2d2.R2D2Config(BATCHSIZE=batch, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=slots, BUFFER_SIZE=0,
                           LEARNER_DEVICE="cuda:0", FRAME_STRIP=True, FRAME_DEDUP=dedup,
                           HOST_POOL=kind == "host_pool", HOST_FRAMES=kind == "host_frames", **kw)


def _block(push_batch):
    strips, a, r, h0, h1, nd, _ = player_sequences(BLOCK, T=T, actors=32, episode=(800, 2400), seed=1)
    p = (np.random.default_rng(2).random(BLOCK) + 0.05).astype(np.float32)
    out = []
    for i in range(0, BLOCK, push_batch):
        chunk = []
        for x in (strips, a, r, h0, h1, nd, p):
            t = torch.from_numpy(np.ascontiguousarray(x[i:i + push_batch]))
            pin = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
            pin.copy_(t)
            chunk.append(pin)
        out.append(chunk)
    return out


def _fill(memory, block, n) -> float:
    """Push n sequences (the block, repeated); -> sequences/s."""
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
    """ms per call of fn(i), i < n, by CUDA events."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def in_process(block, seqs, batch, steps, rounds, warmup) -> dict:
    learners, res = {}, {"push_sequences_per_s": {}, "fused_step_per_s": {k: [] for k in KINDS}}
    for kind in KINDS:
        torch.manual_seed(0)
        L = r2d2.Learner(_cfg(kind, seqs, batch), start_replay=False)
        res["push_sequences_per_s"][kind] = round(_fill(L.memory, block, seqs))
        L.memory.store.seed(7, 0)
        for _ in range(warmup):
            L.fused_step(use_graph=True)
        learners[kind] = L
    res["live"] = {k: len(L.memory.store) for k, L in learners.items()}
    for r in range(rounds):
        for kind in (KINDS if r % 2 == 0 else KINDS[::-1]):
            L = learners[kind]
            res["fused_step_per_s"][kind].append(round(1e3 / _events(lambda i: L.fused_step(use_graph=True), steps),
                                                       1))
        print(json.dumps({"round": r, **{k: v[-1] for k, v in res["fused_step_per_s"].items()}}), flush=True)
    res["gather"] = gather_rates(learners["host_pool"].memory.store, learners["host_frames"].memory.store, batch)
    res["serve_fill_ms"] = {k: serve_fill_ms(learners[k].memory.store, batch) for k in ("hbm_pool", "host_pool")}
    for L in learners.values():
        torch.cuda.synchronize()
        L.memory.store.close()
    return res


def gather_rates(pool_store, rows_store, batch, iters=50, rounds=3) -> dict:
    """GB/s of B strips gathered from the host pool (k_gather_host_planes) and from host rows (k_gather_host_rows)."""
    idx = torch.randint(0, len(pool_store), (batch,), device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    outs = {"host_planes": (pool_store, pool_store.alloc_batch(batch, ("state",))),
            "host_rows": (rows_store, rows_store.alloc_batch(batch, ("state",)))}
    res = {k: [] for k in outs}
    for _ in range(rounds):
        for k, (st, out) in outs.items():
            for _ in range(5):
                st.gather(idx, out)
            res[k].append(round(batch * STRIP_BYTES / (_events(lambda i: st.gather(idx, out), iters) / 1e3) / 1e9, 2))
    res["minibatch_bytes"] = batch * STRIP_BYTES
    return res


def serve_fill_ms(st, batch, slots=8, fills=50) -> float:
    ring = ServeRing.create(st, batch, slots)
    for k in range(slots):
        ring.fill(st, k, k + 1, 0.4)
    ms = _events(lambda i: ring.fill(st, i % slots, 100 + i, 0.4), fills)
    torch.cuda.synchronize()
    ring.close()
    return round(ms, 3)


def capacity(block, log2seq, limit) -> dict:
    n = 1 << log2seq
    F, W = r2d2.dedup_geometry(_cfg("host_pool", n, 64))
    pinned = F * R.FRAME_BYTES
    out = {"log2seq": log2seq, "sequences": n, "pool_frames": F, "host_bytes_needed": pinned,
           "host_limit_bytes": limit}
    if pinned > limit:
        out.update(measured=False, reason="the host limit (--max-host-gb, half of MemAvailable) is below the pool")
        return out
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    rp = r2d2.Replay(_cfg("host_pool", n, 64))
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    pushed = n + n // 4
    rate = _fill(rp, block, pushed)                        # past the slot ring's wrap
    st = rp.store
    out.update(measured=True, device_total=total, device_bytes_used_by_store=free0 - free1, host_bytes_pinned=pinned,
               pushed=pushed, live=len(st), head=st.head, head_seq=st.head_seq, push_sequences_per_s=round(rate),
               pool_is_pinned_host=bool(st.pool.is_pinned()))
    st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seqs", type=int, default=1 << 14)
    ap.add_argument("--push-batch", type=int, default=256)
    ap.add_argument("--log2seq", type=int, default=None)
    ap.add_argument("--max-host-gb", type=float, default=200.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    limit = host_limit(a.max_host_gb)
    res = {"gpu": _card(), "batch": a.batch, "seqs": a.seqs, "host_limit_bytes": limit}
    print(json.dumps(res), flush=True)
    block = _block(a.push_batch)
    res.update(in_process(block, a.seqs, a.batch, a.steps, a.rounds, a.warmup))
    gc.collect()
    torch.cuda.empty_cache()
    log2seq = a.log2seq
    if log2seq is None:
        log2seq = 17
        per_seq = r2d2.R2D2Config.FRAMES_PER_SEQUENCE * R.FRAME_BYTES
        while log2seq < 20 and (2 << log2seq) * per_seq <= limit:
            log2seq += 1
    res["capacity"] = capacity(block, log2seq, limit)
    res["fused_step_range"] = {k: [min(v), max(v)] for k, v in res["fused_step_per_s"].items()}
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_r2d2_host_pool.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
