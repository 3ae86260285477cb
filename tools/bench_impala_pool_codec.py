"""Coded IMPALA frame pool (ImpalaConfig.STAGED_POOL_CODEC) against the raw frame-deduplicated store (FRAME_DEDUP), on
one GPU.

    python tools/bench_impala_pool_codec.py [--batch 32 1024] [--slots 2048] [--steps 50] [--rounds 3]

Rollouts are synthetic: the reference IMPALA actors' structure (tests/impala_rollouts.py, IMPALA/Player.py: stacks of
the last four frames, the bootstrap stack, checkLength's padding, --actors actors interleaved) over the synthetic
Atari-like frames of tests/pool_codec_model.py (tests/impala_atari_rollouts.py).  No real Atari frame is used, so the
bytes per frame below are those of synthetic frames.  Prints one JSON line with
  * bytes stored per distinct frame (codec_stats) and distinct frames staged per drawn rollout;
  * push_arrays rollouts/s from pinned host buffers, raw and coded;
  * the captured in-process fused_step at each --batch, raw and coded, alternating (--rounds rounds each);
  * the staging kernel (b2rl_dedup_stage_rollouts) at each --batch, by CUDA events over many launches;
  * b2rl_serve_fill_uniform fills/s at each --batch, raw and coded, alternating;
  * the device memory taken by creating (not filling) coded stores of --big-slots rollouts (torch.cuda.mem_get_info),
    their rings sized at 1.25 x the measured ring bytes per rollout (new frames x bytes per frame), and the default
    ring at the smallest of them.
The GPU's name, power limit and maximum SM clock are part of the output."""
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
from distributed_rl_b200 import impala, replay as R  # noqa: E402
from distributed_rl_b200.replay_server import ServeRing  # noqa: E402
from impala_atari_rollouts import atari_rollouts  # noqa: E402

T = 20
NAMES = ("raw", "coded")


def _pinned(xs):
    out = []
    for x in xs:
        t = torch.from_numpy(x)
        p = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        p.copy_(t)
        out.append(p)
    return out


def _cfg(name, slots, batch, **kw):
    return impala.ImpalaConfig(BATCHSIZE=batch, UNROLL_STEP=T, REPLAY_MEMORY_LEN=slots, BUFFER_SIZE=0,
                               LEARNER_DEVICE="cuda:0", FRAME_DEDUP=True, STAGED_POOL_CODEC=name == "coded",
                               DEDUP_WINDOW=4096, **kw)


def _timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    e1.synchronize()
    return n / (e0.elapsed_time(e1) / 1e3)


def _steps(steps, batch):
    return max(5, steps * 32 // batch)


def ingest(rollouts, slots, push_batch):
    """-> push rates, bytes per frame and per slot, and the two replays (filled)."""
    n = rollouts[0].shape[0]
    host = [_pinned([x[i:i + push_batch] for x in rollouts]) for i in range(0, n, push_batch)]
    res = {"push_rollouts_per_s": {}}
    replays = {}
    for name in NAMES:
        rp = impala.Replay(_cfg(name, slots, 32))
        rp.push_arrays(*host[0])                                       # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for h in host[1:]:
            rp.push_arrays(*h)
        torch.cuda.synchronize()
        res["push_rollouts_per_s"][name] = round(push_batch * (len(host) - 1) / (time.perf_counter() - t0))
        replays[name] = rp
    st = replays["coded"].store
    s = st.codec_stats()
    new = st.head_seq / n
    small = sum(f.nbytes for f in st.fields)
    res.update(live=len(st), pool_frames=st.pool_frames, window=st.window, new_frames_per_rollout=round(new, 2),
               bytes_per_frame=round(s["bytes_per_frame"], 1), raw_bytes_per_frame=R.FRAME_BYTES,
               coded_bytes_per_slot=round(new * s["bytes_per_frame"] + small),
               raw_bytes_per_slot=round(new * R.FRAME_BYTES + small))
    return res, replays


def staging(store, batch, steps):
    """Distinct frames staged per drawn rollout, and the staging kernel's time by CUDA events."""
    out = {"idx": torch.empty(batch, dtype=torch.int64, device="cuda")}
    store.seed(5, 0)
    store.uniform_fetch(batch, T, out)
    staged = store.alloc_staged(batch)
    store.stage_frames(out["idx"], staged)
    Rf = 4 * (T + 1)
    first = staged["planes"] == torch.arange(batch * Rf, device="cuda", dtype=torch.int32).view(batch, Rf)
    distinct = first.sum().item() / batch
    n = max(20, 20 * steps * 32 // batch)
    rate = _timed(lambda i: store.stage_frames(out["idx"], staged), n)
    del staged
    return {"distinct_frames_per_rollout": round(distinct, 2), "stage_us": round(1e6 / rate, 1),
            "staged_frames_per_s": round(distinct * batch * rate)}


def captured_steps(replays, slots, batch, steps, rounds):
    learners = {}
    for name in NAMES:
        torch.manual_seed(0)
        L = impala.Learner(_cfg(name, slots, batch), start_replay=False, memory=None)
        L._memory = replays[name]                                      # the filled replay, shared across batch sizes
        replays[name].store.seed(7, 0)
        L.fused_step(use_graph=True)
        learners[name] = L
    out = {name: [] for name in NAMES}
    n = _steps(steps, batch)
    for _ in range(rounds):
        for name, L in learners.items():
            out[name].append(round(_timed(lambda i: L.fused_step(use_graph=True), n), 1))
    del learners
    gc.collect()
    torch.cuda.empty_cache()
    return out


def fills(replays, batch, steps, rounds, ring_slots=4):
    rings = {}
    for name in NAMES:
        st = replays[name].store
        st.seed(9, 0)
        ring = ServeRing.create(st, batch, ring_slots)
        for k in range(ring_slots):
            ring.fill_uniform(st, k, k + 1, T)
        rings[name] = (st, ring)
    out = {name: [] for name in NAMES}
    n = 4 * _steps(steps, batch)
    for _ in range(rounds):
        for name, (st, ring) in rings.items():
            out[name].append(round(_timed(lambda i: ring.fill_uniform(st, i % ring_slots, i + 100, T), n), 1))
    torch.cuda.synchronize()
    for _, ring in rings.values():
        ring.close()
    return out


def big_store_memory(slots, bytes_per_rollout):
    """Device memory of creating a coded store of `slots` rollouts with POOL_BYTES_PER_ROLLOUT = bytes_per_rollout
    (None: the default ring, (F + 1) x 7 072 bytes)."""
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    cfg = impala.ImpalaConfig(REPLAY_MEMORY_LEN=slots, FRAME_DEDUP=True, STAGED_POOL_CODEC=True,
                              POOL_BYTES_PER_ROLLOUT=bytes_per_rollout)
    F, W = impala.dedup_geometry(cfg)
    pb = impala.pool_bytes(cfg)
    st = R.RolloutDedupReplay(slots, F, W, T=T, pool_bytes=pb)
    free1, _ = torch.cuda.mem_get_info()
    out = {"slots": slots, "pool_frames": F, "window": W, "pool_bytes_per_rollout": bytes_per_rollout,
           "ring_GB": round(pb / 1e9, 2), "store_GB": round((free0 - free1) / 1e9, 2),
           "raw_dedup_pool_GB": round(F * R.FRAME_BYTES / 1e9, 2), "card_GB": round(total / 1e9, 2)}
    st.close()
    del st
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[32, 1024])
    ap.add_argument("--slots", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--actors", type=int, default=32)
    ap.add_argument("--episode", type=int, nargs=2, default=(200, 800))
    ap.add_argument("--p-done", type=float, default=0.01)
    ap.add_argument("--push-batch", type=int, default=256)
    ap.add_argument("--big-slots", type=int, nargs="*", default=[100_000, 1_000_000])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_impala_pool_codec measures the GPU store: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    state, act, mu, rew, done, kind = atari_rollouts(a.slots, T=T, actors=a.actors, episode=tuple(a.episode),
                                                     p_done=a.p_done, seed=1)
    res = {"gpu": gpu, "frames": "synthetic Atari-like (tests/pool_codec_model.atari_frame)", "slots": a.slots,
           "actors": a.actors, "episode": list(a.episode), "p_done": a.p_done,
           "padded_rollouts": kind.count("padded")}
    part, replays = ingest((state, act, mu, rew, done), a.slots, a.push_batch)
    res.update(part)
    del state
    gc.collect()
    res["staging"] = {str(b): staging(replays["coded"].store, b, a.steps) for b in a.batch}
    res["fused_step_per_s"] = {str(b): captured_steps(replays, a.slots, b, a.steps, a.rounds) for b in a.batch}
    res["fill_per_s"] = {str(b): fills(replays, b, a.steps, a.rounds) for b in a.batch}
    for rp in replays.values():
        rp.store.close()
    del replays
    gc.collect()
    torch.cuda.empty_cache()
    per_rollout = round(1.25 * part["new_frames_per_rollout"] * part["bytes_per_frame"])   # the ring's share of a slot
    res["big_store"] = [big_store_memory(s, per_rollout) for s in a.big_slots]
    if a.big_slots:
        res["big_store"].append(big_store_memory(min(a.big_slots), None))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
