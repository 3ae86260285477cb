"""Actor-record ingest on one GPU: Replay.push_records decoding on the device (wire.WireIngest, DESIGN.md §4.24) against
the host decoders (pickle.loads + wire.decode_*), and the captured learner step's rate while an ingest thread pushes
records at a fixed rate on each path.

    python tools/bench_wire_ingest.py [--out DIR]

Prints one JSON line (and writes it to DIR/bench_wire_ingest.json), with the card's name and power limit read in the
same run."""
from __future__ import annotations

import argparse
import json
import os
import pickle
import subprocess
import sys
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from distributed_rl_b200 import apex, impala, r2d2  # noqa: E402


def _gpu() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"gpu": q[0] if q else torch.cuda.get_device_name(), "torch_name": torch.cuda.get_device_name()}


def _records(kind, n, T, rng):
    """Records pickled as the reference Players pickle them (protocol 4, their dtypes)."""
    out = []
    for i in range(n):
        if kind == "apex":
            rec = [rng.integers(0, 256, (4, 84, 84), dtype=np.uint8), int(rng.integers(6)), float(rng.standard_normal()),
                   rng.integers(0, 256, (4, 84, 84), dtype=np.uint8), bool(rng.random() < .02), float(rng.random())]
        elif kind == "r2d2":
            frames = rng.integers(0, 256, (T + 3, 84, 84), dtype=np.uint8)
            rec = [(torch.from_numpy(rng.standard_normal((1, 1, 512)).astype(np.float32)),
                    torch.from_numpy(rng.standard_normal((1, 1, 512)).astype(np.float32)))]
            for t in range(T):
                rec += [frames[t:t + 4].copy(), int(rng.integers(6)), float(rng.standard_normal())]
            rec.append(False)
            arr = np.empty(len(rec), object)
            for j, x in enumerate(rec):
                arr[j] = x
            rec = np.append(arr, float(rng.random()))
        else:
            rec = [rng.integers(0, 256, (T + 1, 28224), dtype=np.uint8), rng.integers(0, 6, (T, 1)),
                   rng.uniform(0.05, 0.9, (T, 1)).astype(np.float32), rng.standard_normal(T), 1]
        out.append(pickle.dumps(rec))
    return out


def _replay(kind, cap, **kw):
    if kind == "apex":
        return apex.Replay(apex.ApexConfig(REPLAY_MEMORY_LEN=cap, BUFFER_SIZE=0, **kw))
    if kind == "r2d2":
        return r2d2.Replay(r2d2.R2D2Config(REPLAY_MEMORY_LEN=cap, BUFFER_SIZE=0, FRAME_STRIP=True, **kw))
    return impala.Replay(impala.ImpalaConfig(REPLAY_MEMORY_LEN=cap, BUFFER_SIZE=0, **kw))


def push_rate(kind, batch, reps, T) -> dict:
    rng = np.random.default_rng(0)
    blobs = _records(kind, batch, T, rng)
    res = {"record_bytes": len(blobs[0]), "batch": batch}
    for path in ("device", "host"):
        rp = _replay(kind, 4 * batch)
        if path == "host":
            rp._wire_decode = lambda b: None
        rp.push_records(blobs)                              # warm-up: template, staging, allocations
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            rp.push_records(blobs)
        torch.cuda.synchronize()
        res[f"{path}_records_per_s"] = round(batch * reps / (time.perf_counter() - t0), 1)
        if path == "device":
            res["host_fallback_records"] = rp._wire.host_records
    return res


def step_rate_under_ingest(kind, rate, seconds, steps_warm=5) -> dict:
    """Captured fused steps per second (CUDA events) while a thread calls push_records at `rate` records/s."""
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(1)
    out = {"ingest_records_per_s_target": rate}
    for path in ("device", "host"):
        if kind == "apex":
            cfg = apex.ApexConfig(BATCHSIZE=512, REPLAY_MEMORY_LEN=1 << 17, BUFFER_SIZE=0, LEARNER_DEVICE=str(dev))
            L = apex.Learner(cfg, connect=None, start_replay=False)
            rp = L.memory
            st = rp.store
            st.fill_hash(cfg.REPLAY_MEMORY_LEN, seed=0xB200)
            st.build(torch.rand(cfg.REPLAY_MEMORY_LEN, device=dev) + 1e-3)
            st.seed(1234, 0)
            blobs, chunk = _records("apex", 64, 0, rng), 64
        else:
            T = 20
            cfg = impala.ImpalaConfig(BATCHSIZE=32, REPLAY_MEMORY_LEN=4096, BUFFER_SIZE=0, UNROLL_STEP=T,
                                      LEARNER_DEVICE=str(dev))
            L = impala.Learner(cfg, connect=None, start_replay=False)
            rp = L._memory
            st = rp.store
            st.fill_hash(cfg.REPLAY_MEMORY_LEN, seed=0xB204)
            st.field_view("action").random_(0, 6)
            st.field_view("mu").uniform_(0.05, 0.9)
            st.field_view("done").fill_(1.0)
            st.build(torch.ones(cfg.REPLAY_MEMORY_LEN, device=dev))
            blobs, chunk = _records("impala", 8, T, rng), 8
        if path == "host":
            rp._wire_decode = lambda b: None
        for _ in range(steps_warm):
            L.fused_step()
        rp.push_records(blobs)
        torch.cuda.synchronize()
        stop, pushed = threading.Event(), [0]

        def ingest():
            t0 = time.perf_counter()
            while not stop.is_set():
                due = t0 + (pushed[0] + chunk) / rate
                if time.perf_counter() < due:
                    time.sleep(min(0.001, due - time.perf_counter()))
                    continue
                rp.push_records(blobs)
                pushed[0] += chunk
        th = threading.Thread(target=ingest, daemon=True)
        th.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        steps, t0 = 0, time.perf_counter()
        e0.record()
        while time.perf_counter() - t0 < seconds:
            L.fused_step()
            steps += 1
        e1.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        stop.set()
        th.join()
        torch.cuda.synchronize()
        out[f"{path}_steps_per_s"] = round(steps / (e0.elapsed_time(e1) / 1e3), 1)
        out[f"{path}_ingest_records_per_s"] = round(pushed[0] / wall, 1)
        del L, rp, st
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=6.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wire_ingest measures on a GPU; none is visible")
    res = _gpu()
    res["push_records"] = {"apex": push_rate("apex", 1024, args.reps, 0),
                           "r2d2_T80_strips": push_rate("r2d2", 32, args.reps, 80),
                           "impala_T20": push_rate("impala", 128, args.reps, 20)}
    res["step_under_ingest"] = {"apex_B512": step_rate_under_ingest("apex", 5000, args.seconds),
                                "impala_B32": step_rate_under_ingest("impala", 800, args.seconds)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_wire_ingest.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
