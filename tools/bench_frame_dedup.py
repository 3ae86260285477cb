"""Frame-deduplicated Ape-X store (ApexConfig.FRAME_DEDUP) against the stack store, on one GPU.

    python tools/bench_frame_dedup.py [--batch 512] [--slots 131072] [--steps 200] [--big-slots 2097152]

Records are generated on the device the way the reference actors make them (APE_X/Player.py): episodes of random
frames, each step's stack the last four frames (an episode starts with its first frame four times), get_traj pairing
stack t with stack t + 3, and 8 actors interleaved 5 records at a time.  Prints one JSON line with
  * ingest records/s from pinned host buffers (push), dedup and stacks, and the new frames per record;
  * the captured fused_step rate, dedup and stacks, alternating (3 rounds each);
  * served: b2rl_serve_fill launches/s into a serve ring created in this process, and the captured bound step
    (SERVED_FUSED_STEP) on slots filled from each store, dedup and stacks, alternating;
  * the device memory of a --big-slots dedup store filled until its slot ring has wrapped.
The GPU's name and power limit are part of the output.  Pushes and learner steps are timed separately: a push
synchronizes its stream once, and its cost to a learner stepping on the same stream is not measured here."""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributed_rl_b200 import apex, replay as R  # noqa: E402
from distributed_rl_b200.replay_server import ServeRing  # noqa: E402


class PlayerStream:
    """Device-side generator of Player-like records for `actors` actors (see the module docstring)."""

    def __init__(self, device, actors=8, episode=200, unroll=3, chunk=5, seed=0):
        self.dev, self.actors, self.E, self.U, self.chunk = device, actors, episode, unroll, chunk
        self.g = torch.Generator(device=device)
        self.g.manual_seed(seed)
        t = torch.arange(episode, device=device)
        self.stack_idx = (t[:, None] - 3 + torch.arange(4, device=device)).clamp_(min=0)      # (E, 4)
        self.next_t = (t + unroll).clamp_(max=episode - 1)
        self.eps = [None] * actors
        self.pos = [episode] * actors
        self.k = 0

    def _take(self, a, m):
        if self.pos[a] >= self.E:
            self.eps[a] = torch.randint(0, 256, (self.E, 84, 84), device=self.dev, dtype=torch.uint8, generator=self.g)
            self.pos[a] = 0
        t = torch.arange(self.pos[a], min(self.E, self.pos[a] + m), device=self.dev)
        self.pos[a] += t.numel()
        f = self.eps[a]
        return f[self.stack_idx[t]], f[self.stack_idx[self.next_t[t]]], (self.next_t[t] == self.E - 1).to(torch.uint8)

    def batch(self, n):
        s, ns, d = [], [], []
        got = 0
        while got < n:
            a, b, c = self._take(self.k, min(self.chunk, n - got))
            s.append(a); ns.append(b); d.append(c)
            got += a.shape[0]
            self.k = (self.k + 1) % self.actors
        act = torch.randint(0, 6, (n,), device=self.dev, dtype=torch.int32, generator=self.g)
        rew = torch.randn(n, device=self.dev, generator=self.g)
        prio = torch.rand(n, device=self.dev, generator=self.g) + 0.01
        return [torch.cat(s), torch.cat(ns), act, rew, torch.cat(d)], prio


def _pinned(xs):
    out = []
    for x in xs:
        p = torch.empty(x.shape, dtype=x.dtype, pin_memory=True)
        p.copy_(x)
        out.append(p)
    return out


def ingest_rate(dev, slots, batch, records):
    gen = PlayerStream(dev, seed=1)
    host = []
    for _ in range(records // batch):
        f, p = gen.batch(batch)
        host.append((_pinned(f), _pinned([p])[0]))
    res = {}
    for name in ("stacks", "dedup"):
        st = (R.DedupReplay(slots, 4 * slots, min(1 << 20, slots // 2), device=dev) if name == "dedup"
              else R.DeviceReplay(slots, R.APEX_FIELDS, dev))
        st.push(*host[0])                                            # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f, p in host[1:]:
            st.push(f, p)
        torch.cuda.synchronize()
        res[name] = round(batch * (len(host) - 1) / (time.perf_counter() - t0))
        if name == "dedup":
            res["new_frames_per_record"] = round(st.head_seq / (batch * len(host)), 3)
        st.close()
    return res


def step_rate(dev, slots, batch, steps, rounds=3):
    learners = {}
    for name in ("stacks", "dedup"):
        cfg = apex.ApexConfig(BATCHSIZE=batch, REPLAY_MEMORY_LEN=slots, BUFFER_SIZE=0, LEARNER_DEVICE=str(dev),
                              FRAME_DEDUP=name == "dedup")
        torch.manual_seed(0)
        L = apex.Learner(cfg, connect=None, start_replay=False)
        gen = PlayerStream(dev, seed=2)
        for _ in range(slots // 4096 + 1):
            f, p = gen.batch(4096)
            L.memory.push_arrays(*f, p)
        L.memory.store.seed(7, 0)
        L.fused_step(use_graph=True)
        learners[name] = L
    rates = {k: [] for k in learners}
    for _ in range(rounds):
        for name, L in learners.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                L.fused_step(use_graph=True)
            e1.record()
            e1.synchronize()
            rates[name].append(steps / (e0.elapsed_time(e1) / 1e3))
    return {k: [round(v, 1) for v in r] for k, r in rates.items()}


def served_rate(dev, slots, batch, steps, rounds=3, ring_slots=16):
    """-> {"fill_per_s": {...}, "bound_step_per_s": {...}} for both stores, alternating."""
    from types import SimpleNamespace
    setups = {}
    for name in ("stacks", "dedup"):
        st = (R.DedupReplay(slots, 4 * slots, min(1 << 20, slots // 8), device=dev) if name == "dedup"
              else R.DeviceReplay(slots, R.APEX_FIELDS, dev))
        gen = PlayerStream(dev, seed=4)
        for _ in range(slots // 4096 + 1):
            f, p = gen.batch(4096)
            st.push(f, p)
        st.seed(9, 0)
        ring = ServeRing.create(st, batch, ring_slots)
        for k in range(ring_slots):
            ring.fill(st, k, k + 1, 0.4)
        torch.manual_seed(0)
        mem = SimpleNamespace(ring=ring, acquire=None, release=None, is_alive=lambda: True)
        L = apex.Learner(apex.ApexConfig(BATCHSIZE=batch, REPLAY_MEMORY_LEN=8, BUFFER_SIZE=0, LEARNER_DEVICE=str(dev),
                                         SERVED_FUSED_STEP=True), start_replay=False, memory=mem)
        s = L._fused_state()
        k = [0]

        def step(ring=ring, L=L, s=s, k=k):
            ring.bind(ring.slot_ptrs(k[0] % ring_slots)[0][0], R.APEX_FIELDS, s.cur, s.frames,
                      torch.cuda.current_stream())
            L.fused_step(use_graph=True)
            k[0] += 1
        for _ in range(5):
            step()
        setups[name] = (st, ring, step)
    out = {"fill_per_s": {k: [] for k in setups}, "bound_step_per_s": {k: [] for k in setups}}
    for _ in range(rounds):
        for name, (st, ring, step) in setups.items():
            for key, fn in (("fill_per_s", lambda i: ring.fill(st, i % ring_slots, i + 100, 0.4)),
                            ("bound_step_per_s", lambda i: step())):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(steps):
                    fn(i)
                e1.record()
                e1.synchronize()
                out[key][name].append(round(steps / (e0.elapsed_time(e1) / 1e3), 1))
    for st, ring, _ in setups.values():
        torch.cuda.synchronize()
        ring.close()
    return out


def big_store_memory(dev, slots):
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info(dev)
    cfg = apex.ApexConfig(REPLAY_MEMORY_LEN=slots)
    F, W = apex.dedup_geometry(cfg)
    st = R.DedupReplay(slots, F, W, device=dev)
    free1, _ = torch.cuda.mem_get_info(dev)
    gen = PlayerStream(dev, seed=3)
    pushed, b = 0, st.max_batch
    t0 = time.perf_counter()
    while pushed < slots + b:
        f, p = gen.batch(b)
        st.push(f, p)
        pushed += b
    torch.cuda.synchronize()
    out = {"slots": slots, "pool_frames": F, "window": W, "pool_GB": round(F * R.FRAME_BYTES / 1e9, 2),
           "store_GB": round((free0 - free1) / 1e9, 2), "card_GB": round(total / 1e9, 2), "records_pushed": pushed,
           "live": len(st), "new_frames_per_record": round(st.head_seq / pushed, 3),
           "fill_records_per_s": round(pushed / (time.perf_counter() - t0))}
    st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--slots", type=int, default=1 << 17)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--ingest-batch", type=int, default=1024)
    ap.add_argument("--ingest-records", type=int, default=16384)
    ap.add_argument("--big-slots", type=int, default=1 << 21)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_frame_dedup measures the GPU store: no CUDA device")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "batch": a.batch, "slots": a.slots,
           "ingest_records_per_s": ingest_rate(dev, a.slots, a.ingest_batch, a.ingest_records),
           "fused_step_per_s": step_rate(dev, a.slots, a.batch, a.steps),
           "served": served_rate(dev, a.slots, a.batch, a.steps)}
    gc.collect()                      # the learners' replays (their views reference them) before the big store
    torch.cuda.empty_cache()
    if a.big_slots:
        res["big_store"] = big_store_memory(dev, a.big_slots)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
