"""Frame-deduplicated R2D2 store (R2D2Config.FRAME_DEDUP) against the frame-strip store (FRAME_STRIP), on one GPU.

    python tools/bench_r2d2_frame_dedup.py [--batch 64] [--slots 2048] [--steps 100] [--big-slots 200000]

Sequences are generated on the host the way the reference R2D2 actors send them (tests/strip_dedup_model.py,
R2D2/Player.py): --actors actors (32, the N of cfg/r2d2.json) interleaved, episodes of --episode random frames whose
first stack is the first frame four times, get_traj cutting T = 80 stacks once the buffer holds 128 and dropping 40,
the done sequence being the episode's last 80 stacks.  Prints one JSON line with
  * new frames per sequence and bytes per sequence of the dedup store (pool frames stored + its slot fields);
  * push_arrays sequences/s from pinned host buffers, dedup and strips;
  * the captured in-process fused_step at --batch, dedup and strips, alternating (3 rounds each);
  * the captured served step (SERVED_FUSED_STEP) on ring slots filled from each store, and the fill, alternating;
  * the device memory a --big-slots dedup store takes at the default geometry (torch.cuda.mem_get_info), allocated
    but not filled.
The GPU's name and power limit are part of the output."""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from distributed_rl_b200 import r2d2, replay as R  # noqa: E402
from distributed_rl_b200.replay_server import ServeRing  # noqa: E402
from strip_dedup_model import player_sequences  # noqa: E402

T = 80


def _pinned(xs):
    out = []
    for x in xs:
        t = torch.from_numpy(x)
        p = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        p.copy_(t)
        out.append(p)
    return out


def _cfg(name, slots, batch, **kw):
    return r2d2.R2D2Config(BATCHSIZE=batch, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=slots, BUFFER_SIZE=0,
                           LEARNER_DEVICE="cuda:0", FRAME_STRIP=True, FRAME_DEDUP=name == "dedup", DEDUP_WINDOW=4096,
                           **kw)


def _timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    e1.synchronize()
    return n / (e0.elapsed_time(e1) / 1e3)


def ingest_and_steps(seqs, slots, batch, steps, push_batch, rounds=3):
    """-> ingest rates, new frames and bytes per sequence, and the in-process captured step rates."""
    strips, a, r, h0, h1, nd, _ = seqs
    n = strips.shape[0]
    p = torch.rand(n).numpy() + 0.05
    host = [_pinned([x[i:i + push_batch] for x in (strips, a, r, h0, h1, nd, p)]) for i in range(0, n, push_batch)]
    res = {"push_sequences_per_s": {}, "fused_step_per_s": {}}
    learners = {}
    for name in ("strips", "dedup"):
        torch.manual_seed(0)
        L = r2d2.Learner(_cfg(name, slots, batch), start_replay=False)
        L.memory.push_arrays(*host[0])                                  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for h in host[1:]:
            L.memory.push_arrays(*h)
        torch.cuda.synchronize()
        res["push_sequences_per_s"][name] = round(push_batch * (len(host) - 1) / (time.perf_counter() - t0))
        st = L.memory.store
        if name == "dedup":
            new = st.head_seq / n
            slot = sum(f.nbytes for f in st.fields)
            res.update(live=len(st), pool_frames=st.pool_frames, window=st.window, new_frames_per_sequence=round(new, 2),
                       bytes_per_sequence=round(new * R.FRAME_BYTES + slot), bytes_per_sequence_at_default_pool=round(
                           r2d2.R2D2Config.FRAMES_PER_SEQUENCE * R.FRAME_BYTES + slot),
                       strip_bytes_per_sequence=sum(f.nbytes for f in R.r2d2_fields(T, strip=True)))
        st.seed(7, 0)
        L.fused_step(use_graph=True)
        learners[name] = L
    for name in learners:
        res["fused_step_per_s"][name] = []
    for _ in range(rounds):
        for name, L in learners.items():
            res["fused_step_per_s"][name].append(round(_timed(lambda i: L.fused_step(use_graph=True), steps), 1))
    for L in learners.values():
        L.memory.store.close()
    return res


def served_rate(seqs, slots, batch, steps, rounds=3, ring_slots=8):
    from test_gpu_19_served_sequences import _bind, _local_memory
    strips, a, r, h0, h1, nd, _ = seqs
    n = min(slots, strips.shape[0])
    fields = R.r2d2_fields(T, strip=True)
    setups = {}
    for name in ("strips", "dedup"):
        st = (R.StripDedupReplay(slots, *r2d2.dedup_geometry(_cfg(name, slots, batch)), T=T) if name == "dedup"
              else R.DeviceReplay(slots, fields, "cuda:0"))
        for i in range(0, n, 256):
            st.push([torch.from_numpy(x[i:i + 256]) for x in (strips, a, r, h0, h1, nd)], torch.ones(min(256, n - i)))
        st.seed(9, 0)
        ring = ServeRing.create(st, batch, ring_slots)
        for k in range(ring_slots):
            ring.fill(st, k, k + 1, 0.4)
        torch.manual_seed(0)
        L = r2d2.Learner(_cfg("strips", 8, batch, SERVED_FUSED_STEP=True), start_replay=False,
                         memory=_local_memory(ring))
        s = L._state()
        k = [0]

        def step(ring=ring, L=L, s=s, k=k):
            _bind(ring, k[0] % ring_slots, fields, s)
            L._bound_step()
            k[0] += 1
        for _ in range(5):
            step()
        setups[name] = (st, ring, step)
    out = {"fill_per_s": {k: [] for k in setups}, "bound_step_per_s": {k: [] for k in setups}}
    for _ in range(rounds):
        for name, (st, ring, step) in setups.items():
            out["fill_per_s"][name].append(round(_timed(lambda i: ring.fill(st, i % ring_slots, i + 100, 0.4),
                                                        steps), 1))
            out["bound_step_per_s"][name].append(round(_timed(lambda i: step(), steps), 1))
    for st, ring, _ in setups.values():
        torch.cuda.synchronize()
        ring.close()
        st.close()
    return out


def big_store_memory(slots):
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    F, W = r2d2.dedup_geometry(r2d2.R2D2Config(REPLAY_MEMORY_LEN=slots, FRAME_DEDUP=True))
    st = R.StripDedupReplay(slots, F, W, T=T)
    free1, _ = torch.cuda.mem_get_info()
    out = {"slots": slots, "pool_frames": F, "window": W, "pool_GB": round(F * R.FRAME_BYTES / 1e9, 2),
           "store_GB": round((free0 - free1) / 1e9, 2), "card_GB": round(total / 1e9, 2)}
    st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--slots", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--actors", type=int, default=32)
    ap.add_argument("--episode", type=int, nargs=2, default=(800, 2400))
    ap.add_argument("--push-batch", type=int, default=256)
    ap.add_argument("--big-slots", type=int, default=200_000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_r2d2_frame_dedup measures the GPU store: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    seqs = player_sequences(a.slots, T=T, actors=a.actors, episode=tuple(a.episode), seed=1)
    res = {"gpu": gpu, "batch": a.batch, "slots": a.slots, "actors": a.actors, "episode": list(a.episode)}
    res.update(ingest_and_steps(seqs, a.slots, a.batch, a.steps, a.push_batch))
    gc.collect()
    torch.cuda.empty_cache()
    res["served"] = served_rate(seqs, a.slots, a.batch, a.steps)
    del seqs
    gc.collect()
    torch.cuda.empty_cache()
    if a.big_slots:
        res["big_store"] = big_store_memory(a.big_slots)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
