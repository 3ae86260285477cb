"""R2D2 host frames (R2D2Config.HOST_FRAMES) against frames in HBM, measured in one command.

    python tools/bench_host_frames.py [--batch 64] [--steps 100] [--rounds 3] [--seqs 16384] [--log2seq K]
                                      [--max-host-gb 16] [--out DIR]

Prints one JSON line per measurement and a summary, with the card's name, power limit and maximum SM clock:
  * in-process: steps/s of the captured fused_step at B = 64 over a strip store of --seqs sequences (hash-filled,
    the same contents in both stores), frames in HBM and frames in pinned host memory alternating, --rounds each;
  * served: steps/s of the captured bound step on ring slots filled from a 2048-sequence strip store of each kind,
    and the time of one serve fill (draw + small fields + frames into the slot);
  * gather: GB/s of the host-row gather of a B = 64 strip minibatch (37.5 MB) for a sweep of CTA counts
    (B2RL_HOST_GATHER_CTAS), beside the pinned host-to-device cudaMemcpy rate measured as tools/h2d_probe.py does;
  * push: push_arrays sequences/s of 64 strip sequences from pinned buffers, host store against HBM store;
  * capacity: device memory used (torch.cuda.mem_get_info before and after) and host memory pinned by a strip store of
    2^K sequences, created, hash-filled and stepped three times by the captured fused_step.  K defaults to the largest
    store the host limit allows.
Host memory is shared: no store pins more than --max-host-gb or half of MemAvailable; a store that would is not created
and is reported as not measured.  Needs a GPU; there is no CPU fallback."""
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
STRIP_BYTES = (T + 3) * R.FRAME_BYTES          # 585 648 B of frames per sequence
SWEEP = (1, 2, 4, 8, 12, 16, 24, 32, 48, 66, 132)


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"card": q.stdout.strip() or torch.cuda.get_device_name(0)}


def _meminfo() -> dict:
    out = {}
    with open("/proc/meminfo") as f:
        for line in f:
            k, v = line.split(":")
            if k in ("MemTotal", "MemAvailable"):
                out[k] = int(v.split()[0]) * 1024
    return out


def host_limit(max_host_gb: float) -> int:
    """The most pinned host memory one store may take: --max-host-gb, and half of MemAvailable."""
    return int(min(max_host_gb * 1e9, _meminfo()["MemAvailable"] / 2))


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


def _learner(host: bool, B: int, n: int):
    torch.manual_seed(0)
    L = r2d2.Learner(r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=n, FRAME_STRIP=True,
                                     HOST_FRAMES=host, LEARNER_DEVICE="cuda:0"), start_replay=False)
    _fill(L.memory.store, n, 5)
    L.memory.store.build(torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(5)) + 0.05)
    L.memory.store.seed(1, 0)
    return L


def _free(L):
    torch.cuda.synchronize()
    L.memory.store.close()
    del L
    torch.cuda.empty_cache()


def in_process(host: bool, B: int, n: int, steps: int, warmup: int) -> float:
    L = _learner(host, B, n)
    for _ in range(warmup):
        L.fused_step(use_graph=True)
    rate = _timed(lambda: L.fused_step(use_graph=True), steps)
    _free(L)
    return rate


def served(host: bool, B: int, steps: int, warmup: int) -> tuple:
    fields = R.r2d2_fields(T, strip=True)
    n = 2048
    st = R.DeviceReplay(n, fields, "cuda:0", host_fields=("state",) if host else ())
    _fill(st, n, 7)
    st.build(torch.rand(n, device="cuda") + 0.05)
    st.seed(3, 0)
    slot_rows = 16
    ring = ServeRing.create(st, B, slot_rows)
    for k in range(slot_rows):                                   # warm
        ring.fill(st, k, k + 1, 0.4)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(slot_rows):
        ring.fill(st, k, k + 1, 0.4)
    e1.record()
    torch.cuda.synchronize()
    fill_ms = e0.elapsed_time(e1) / slot_rows
    torch.manual_seed(0)
    mem = SimpleNamespace(ring=ring, acquire=None, release=None, is_alive=lambda: True)
    L = r2d2.Learner(r2d2.R2D2Config(BATCHSIZE=B, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=8, FRAME_STRIP=True,
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
    torch.cuda.synchronize()
    ring.close()
    st.close()
    del L
    torch.cuda.empty_cache()
    return rate, fill_ms


def gather_sweep(B: int, iters: int = 50) -> dict:
    """GB/s of the host-row gather of B strips (random rows of a 2048-sequence host store) per CTA count."""
    n = 2048
    st = R.DeviceReplay(n, (R.Field("state", torch.uint8, (T + 3, 84, 84)),), "cuda:0", host_fields=("state",))
    st.fill_hash(n, seed=11)
    out = st.alloc_batch(B)
    idx = torch.randint(0, n, (B,), device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    res = {}
    saved = os.environ.get("B2RL_HOST_GATHER_CTAS")
    for ctas in SWEEP:
        os.environ["B2RL_HOST_GATHER_CTAS"] = str(ctas)
        for _ in range(5):
            st.gather(idx, out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            st.gather(idx, out)
        e1.record()
        torch.cuda.synchronize()
        res[ctas] = B * STRIP_BYTES * iters / (e0.elapsed_time(e1) / 1e3) / 1e9
    if saved is None:
        os.environ.pop("B2RL_HOST_GATHER_CTAS")
    else:
        os.environ["B2RL_HOST_GATHER_CTAS"] = saved
    ok = torch.equal(out["state"].cpu(), st.field_view("state").index_select(0, idx.cpu()))
    st.close()
    return {"gbps_by_ctas": res, "last_gather_matches_index_select": ok}


def memcpy_rate(nbytes: int, iters: int = 50) -> float:
    """Pinned host -> device cudaMemcpy GB/s of one nbytes buffer (tools/h2d_probe.py's method)."""
    from distributed_rl_b200 import hostmem
    h = hostmem.pinned_empty((nbytes,), torch.uint8, "cuda:0")
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(s):
        for _ in range(10):
            d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        e0.record(s)
        for _ in range(iters):
            d.copy_(h, non_blocking=True)
        e1.record(s)
    torch.cuda.synchronize()
    return nbytes * iters / (e0.elapsed_time(e1) / 1e3) / 1e9


def push_rate(host: bool, n: int, reps: int) -> float:
    cfg = r2d2.R2D2Config(BATCHSIZE=32, FIXED_TRAJECTORY=T, REPLAY_MEMORY_LEN=4 * n, FRAME_STRIP=True,
                          HOST_FRAMES=host, LEARNER_DEVICE="cuda:0")
    rp = r2d2.Replay(cfg)
    cols = [torch.randint(0, 256, (n, T + 3, 84, 84), dtype=torch.uint8).pin_memory(),
            torch.zeros(n, T, dtype=torch.int32).pin_memory(), torch.zeros(n, T).pin_memory(),
            torch.zeros(n, 512).pin_memory(), torch.zeros(n, 512).pin_memory(), torch.ones(n).pin_memory(),
            torch.ones(n).pin_memory()]
    rp.push_arrays(*cols)
    rate = _timed(lambda: rp.push_arrays(*cols), reps) * n
    rp.store.close()
    return rate


def capacity(log2seq: int, limit: int, B: int) -> dict:
    n = 1 << log2seq
    pinned = n * STRIP_BYTES
    out = {"log2seq": log2seq, "sequences": n, "host_bytes_needed": pinned, "host_limit_bytes": limit}
    if pinned > limit:
        out["measured"] = False
        out["reason"] = "the host limit (--max-host-gb, half of MemAvailable) is below the pinned bytes"
        return out
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    t0 = time.perf_counter()
    L = _learner(True, B, n)
    torch.cuda.synchronize()
    t_fill = time.perf_counter() - t0
    free1, _ = torch.cuda.mem_get_info()
    outs = [L.fused_step(use_graph=True) for _ in range(3)]
    torch.cuda.synchronize()
    out.update(measured=True, device_total=total, device_free_before=free0, device_free_after_store=free1,
               device_bytes_used_by_store_and_learner=free0 - free1, host_bytes_pinned=pinned,
               create_fill_build_s=t_fill, steps_finite=bool(torch.isfinite(outs[-1]["prio"]).all()),
               max_idx=int(outs[-1]["idx"].max()))
    _free(L)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seqs", type=int, default=1 << 14)
    ap.add_argument("--log2seq", type=int, default=None)
    ap.add_argument("--max-host-gb", type=float, default=16.0)
    ap.add_argument("--push-n", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    limit = host_limit(a.max_host_gb)
    seqs = a.seqs
    while seqs * STRIP_BYTES > limit:
        seqs //= 2
    res = dict(_card(), **_meminfo(), host_limit_bytes=limit, batch=a.batch, steps=a.steps, rounds=a.rounds,
               seqs=seqs, in_process={"hbm": [], "host": []}, served={"hbm": [], "host": []},
               serve_fill_ms={"hbm": [], "host": []}, push_seq_per_s={"hbm": [], "host": []})
    print(json.dumps({k: res[k] for k in ("card", "MemTotal", "MemAvailable", "host_limit_bytes", "seqs")}), flush=True)
    for r in range(a.rounds):
        for name in ("hbm", "host") if r % 2 == 0 else ("host", "hbm"):
            host = name == "host"
            res["in_process"][name].append(in_process(host, a.batch, seqs, a.steps, a.warmup))
            rate, fill_ms = served(host, a.batch, a.steps, a.warmup)
            res["served"][name].append(rate)
            res["serve_fill_ms"][name].append(fill_ms)
            res["push_seq_per_s"][name].append(push_rate(host, a.push_n, 10))
            print(json.dumps({"round": r, "frames": name, "in_process": res["in_process"][name][-1],
                              "served": rate, "serve_fill_ms": fill_ms, "push": res["push_seq_per_s"][name][-1]}),
                  flush=True)
    res["gather"] = gather_sweep(a.batch)
    res["memcpy_h2d_gbps"] = memcpy_rate(a.batch * STRIP_BYTES)
    print(json.dumps({"gather": res["gather"], "memcpy_h2d_gbps": res["memcpy_h2d_gbps"]}), flush=True)
    log2seq = a.log2seq
    if log2seq is None:
        log2seq = 10
        while log2seq < 20 and (2 << log2seq) * STRIP_BYTES <= limit:
            log2seq += 1
    res["capacity"] = capacity(log2seq, limit, a.batch)
    for key in ("in_process", "served", "push_seq_per_s"):
        res[key + "_range"] = {k: [min(v), max(v)] for k, v in res[key].items()}
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_host_frames.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
