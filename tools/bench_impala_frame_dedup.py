"""Frame-deduplicated IMPALA store (ImpalaConfig.FRAME_DEDUP) against the stack store, on one GPU.

    python tools/bench_impala_frame_dedup.py [--batch 32 1024] [--slots 2048] [--steps 50] [--big-slots 100000]

Rollouts are generated on the host the way the reference IMPALA actors send them (tests/impala_rollouts.py,
IMPALA/Player.py): --actors actors interleaved, episodes of --episode random frames whose first stack is the first
frame four times, T = 20 steps per rollout with the bootstrap stack, a life lost with probability --p-done per step
ending a rollout early, and checkLength padding such a rollout with the previous rollout's stacks.  Prints one JSON line
with
  * new frames per rollout and bytes per slot of the dedup store (pool frames stored + its slot fields), and at the
    default pool of FRAMES_PER_ROLLOUT frames per slot, against a stack store's slot;
  * push_arrays rollouts/s from pinned host buffers, dedup and stacks;
  * the captured in-process fused_step at each --batch, dedup and stacks, alternating (3 rounds each);
  * b2rl_serve_fill_uniform fills/s and the captured served step (SERVED_FUSED_STEP) on ring slots filled from each
    store, alternating;
  * the device memory a --big-slots dedup store takes at the default geometry (torch.cuda.mem_get_info), allocated
    but not filled.
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
from impala_rollouts import player_rollouts  # noqa: E402

T = 20
NAMES = ("stacks", "dedup")


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
                               LEARNER_DEVICE="cuda:0", FRAME_DEDUP=name == "dedup", DEDUP_WINDOW=4096, **kw)


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
    """-> push rates, new frames and bytes per slot, and the two learners' replays (filled)."""
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
        st = rp.store
        if name == "dedup":
            new = st.head_seq / n
            slot = sum(f.nbytes for f in st.fields)
            res.update(live=len(st), pool_frames=st.pool_frames, window=st.window, new_frames_per_rollout=round(new, 2),
                       bytes_per_slot=round(new * R.FRAME_BYTES + slot), bytes_per_slot_at_default_pool=round(
                           impala.ImpalaConfig.FRAMES_PER_ROLLOUT * R.FRAME_BYTES + slot),
                       stack_bytes_per_slot=sum(f.nbytes for f in R.impala_fields(T)))
        replays[name] = rp
    return res, replays


def captured_steps(replays, slots, batch, steps, rounds=3):
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
    return out


def served(replays, batch, steps, rounds=3, ring_slots=4):
    from test_gpu_19_served_sequences import _bind, _local_memory
    fields = R.impala_fields(T)
    setups = {}
    for name in NAMES:
        st = replays[name].store
        st.seed(9, 0)
        ring = ServeRing.create(st, batch, ring_slots)
        for k in range(ring_slots):
            ring.fill_uniform(st, k, k + 1, T)
        torch.manual_seed(0)
        L = impala.Learner(_cfg("stacks", 8, batch, SERVED_FUSED_STEP=True), start_replay=False,
                           memory=_local_memory(ring))
        s = L._bound_state()
        k = [0]

        def step(ring=ring, L=L, s=s, k=k):
            _bind(ring, k[0] % ring_slots, fields, s)
            L._bound_step()
            k[0] += 1
        for _ in range(5):
            step()
        setups[name] = (st, ring, step)
    out = {"fill_per_s": {k: [] for k in setups}, "bound_step_per_s": {k: [] for k in setups}}
    n = _steps(steps, batch)
    for _ in range(rounds):
        for name, (st, ring, step) in setups.items():
            out["fill_per_s"][name].append(round(_timed(lambda i: ring.fill_uniform(st, i % ring_slots, i + 100, T),
                                                        4 * n), 1))
            out["bound_step_per_s"][name].append(round(_timed(lambda i: step(), n), 1))
    for _, ring, _ in setups.values():
        torch.cuda.synchronize()
        ring.close()
    return out


def big_store_memory(slots):
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    F, W = impala.dedup_geometry(impala.ImpalaConfig(REPLAY_MEMORY_LEN=slots, FRAME_DEDUP=True))
    st = R.RolloutDedupReplay(slots, F, W, T=T)
    free1, _ = torch.cuda.mem_get_info()
    out = {"slots": slots, "pool_frames": F, "window": W, "pool_GB": round(F * R.FRAME_BYTES / 1e9, 2),
           "store_GB": round((free0 - free1) / 1e9, 2),
           "stack_store_GB": round(slots * sum(f.nbytes for f in R.impala_fields(T)) / 1e9, 2),
           "card_GB": round(total / 1e9, 2)}
    st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[32, 1024])
    ap.add_argument("--slots", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--actors", type=int, default=32)
    ap.add_argument("--episode", type=int, nargs=2, default=(400, 1600))
    ap.add_argument("--p-done", type=float, default=0.01)
    ap.add_argument("--push-batch", type=int, default=256)
    ap.add_argument("--big-slots", type=int, default=100_000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_impala_frame_dedup measures the GPU store: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    state, act, mu, rew, done, kind = player_rollouts(a.slots, T=T, actors=a.actors, episode=tuple(a.episode),
                                                      p_done=a.p_done, seed=1)
    res = {"gpu": gpu, "slots": a.slots, "actors": a.actors, "episode": list(a.episode), "p_done": a.p_done,
           "padded_rollouts": kind.count("padded")}
    part, replays = ingest((state, act, mu, rew, done), a.slots, a.push_batch)
    res.update(part)
    del state
    gc.collect()
    res["fused_step_per_s"] = {str(b): captured_steps(replays, a.slots, b, a.steps) for b in a.batch}
    res["served"] = {str(b): served(replays, b, a.steps) for b in a.batch}
    for rp in replays.values():
        rp.store.close()
    del replays
    gc.collect()
    torch.cuda.empty_cache()
    if a.big_slots:
        res["big_store"] = big_store_memory(a.big_slots)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
