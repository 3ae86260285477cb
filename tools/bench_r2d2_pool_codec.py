"""The deduplicated R2D2 store with its frames stored encoded (R2D2Config.POOL_CODEC), measured in one command.

    python tools/bench_r2d2_pool_codec.py [--batch 64] [--steps 100] [--rounds 3] [--seqs 16384] [--log2seq 20]

Every frame here is SYNTHETIC: tests/pool_codec_model.py renders Atari-like frames (flat background, walls, bricks,
paddles, a ball, a score) and cuts them into sequences as the reference R2D2 actors do (32 interleaved actors).  There
is no emulator on the machines this runs on, so no ratio below is a ratio on real Atari frames.  The stores are filled
by pushing one block of 2048 such sequences from pinned buffers, over and over (a copy older than the dedup window is
stored again).  Prints, with the card's name, power limit and maximum SM clock:
  * bytes per stored frame: b2rl_frame_encode on the block's frames and on uniformly random frames, and the coded
    store's codec_stats() after it is filled;
  * in-process: steps/s of the captured fused_step at B = --batch over --seqs sequences, on a plain FRAME_DEDUP store
    ("plain") and a POOL_CODEC store ("coded"), alternating, --rounds rounds each;
  * push: push_arrays sequences/s from pinned buffers while those stores are filled;
  * decode: GB/s of the decode-assemble gather (k_decode_planes: B strips, B (T + 3) 7 056 bytes out);
  * serve fill: ms of one b2rl_serve_fill from each store;
  * capacity: a POOL_CODEC store of 2^--log2seq sequences, POOL_BYTES_PER_SEQUENCE set from the units per sequence
    measured above (with --margin), filled past its slot ring's and unit ring's wraps: device bytes
    (torch.cuda.mem_get_info) and live slots.
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

from distributed_rl_b200 import r2d2, replay as R  # noqa: E402
from distributed_rl_b200.replay_server import ServeRing  # noqa: E402
from pool_codec_model import atari_sequences  # noqa: E402

T = 80
BLOCK = 2048
STRIP_BYTES = (T + 3) * R.FRAME_BYTES
KINDS = ("plain", "coded")


def _card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _cfg(kind, slots, batch, **kw):
    return r2d2.R2D2Config(BATCHSIZE=batch, FIXED_TRAJECTORY=T, MEM=20, REPLAY_MEMORY_LEN=slots, BUFFER_SIZE=0,
                           LEARNER_DEVICE="cuda:0", FRAME_DEDUP=True, POOL_CODEC=kind == "coded", **kw)


def _block(push_batch):
    strips, a, r, h0, h1, nd, _ = atari_sequences(BLOCK, T=T, actors=32, episode=(800, 2400), seed=1)
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
    return out, strips


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


def frame_sizes(strips) -> dict:
    """Mean encoded bytes per frame (b2rl_frame_encode) of the block's distinct frames and of random frames."""
    frames = np.unique(strips.reshape(-1, R.FRAME_BYTES), axis=0)[:20000]
    _, units = R.encode_frames(torch.from_numpy(frames).cuda())
    rnd = torch.randint(0, 256, (2048, 84, 84), dtype=torch.uint8, device="cuda",
                        generator=torch.Generator("cuda").manual_seed(5))
    _, ru = R.encode_frames(rnd)
    u = units.double().cpu()
    return {"synthetic_frames": len(frames), "synthetic_bytes_per_frame": round(16 * float(u.mean()), 1),
            "synthetic_bytes_max": int(16 * u.max()), "synthetic_ratio": round(R.FRAME_BYTES / (16 * float(u.mean())), 2),
            "random_bytes_per_frame": round(16 * float(ru.double().mean()), 1)}


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
    st = learners["coded"].memory.store
    res["codec_stats"] = dict(st.codec_stats(), sequences_pushed=seqs)
    res["live"] = {k: len(L.memory.store) for k, L in learners.items()}
    for r in range(rounds):
        for kind in (KINDS if r % 2 == 0 else KINDS[::-1]):
            L = learners[kind]
            res["fused_step_per_s"][kind].append(round(1e3 / _events(lambda i: L.fused_step(use_graph=True), steps),
                                                       1))
        print(json.dumps({"round": r, **{k: v[-1] for k, v in res["fused_step_per_s"].items()}}), flush=True)
    res["decode_gbs"] = decode_rate(st, batch)
    res["serve_fill_ms"] = {k: serve_fill_ms(L.memory.store, batch) for k, L in learners.items()}
    for L in learners.values():
        torch.cuda.synchronize()
        L.memory.store.close()
    return res


def decode_rate(st, batch, iters=50, rounds=3) -> dict:
    """GB/s written by the decode-assemble gather of B strips (the bytes of B raw strips over its time)."""
    idx = torch.randint(0, len(st), (batch,), device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    out = st.alloc_batch(batch, ("state",))
    res = []
    for _ in range(rounds):
        for _ in range(5):
            st.gather(idx, out)
        res.append(round(batch * STRIP_BYTES / (_events(lambda i: st.gather(idx, out), iters) / 1e3) / 1e9, 2))
    return {"gbs": res, "minibatch_bytes": batch * STRIP_BYTES}


def serve_fill_ms(st, batch, slots=8, fills=50) -> float:
    ring = ServeRing.create(st, batch, slots)
    for k in range(slots):
        ring.fill(st, k, k + 1, 0.4)
    ms = _events(lambda i: ring.fill(st, i % slots, 100 + i, 0.4), fills)
    torch.cuda.synchronize()
    ring.close()
    return round(ms, 3)


def capacity(block, log2seq, bytes_per_seq) -> dict:
    n = 1 << log2seq
    cfg = _cfg("coded", n, 64, POOL_BYTES_PER_SEQUENCE=bytes_per_seq)
    F, W = r2d2.dedup_geometry(cfg)
    out = {"log2seq": log2seq, "sequences": n, "pool_frames": F, "window": W, "pool_bytes_per_sequence": bytes_per_seq,
           "pool_bytes": r2d2.pool_bytes(cfg)}
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    rp = r2d2.Replay(cfg)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    pushed = n + n // 2
    rate = _fill(rp, block, pushed)                        # past the slot ring's and the unit ring's wraps
    st = rp.store
    free2, _ = torch.cuda.mem_get_info()
    out.update(device_total=total, device_bytes_used_by_store=free0 - free1, device_free_after_fill=free2,
               pushed=pushed, live=len(st), head=st.head, head_seq=st.head_seq, push_sequences_per_s=round(rate),
               codec_stats=st.codec_stats())
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
    ap.add_argument("--log2seq", type=int, default=20)
    ap.add_argument("--margin", type=float, default=1.25)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res = {"gpu": _card(), "batch": a.batch, "seqs": a.seqs, "frames": "synthetic Atari-like (tests/pool_codec_model.py)"}
    print(json.dumps(res), flush=True)
    block, strips = _block(a.push_batch)
    res["frame_sizes"] = frame_sizes(strips)
    print(json.dumps(res["frame_sizes"]), flush=True)
    res.update(in_process(block, a.seqs, a.batch, a.steps, a.rounds, a.warmup))
    gc.collect()
    torch.cuda.empty_cache()
    cs = res["codec_stats"]
    # the slot ring must wrap before the byte rule kills: P - 7072 (W + 1) >= N x the bytes a sequence adds
    W = r2d2.R2D2Config.DEDUP_WINDOW
    per_seq = 16.0 * cs["units_written"] / cs["sequences_pushed"]
    bytes_per_seq = round(a.margin * per_seq + 7072 * (W + 1) / (1 << a.log2seq), 1)
    res["capacity"] = capacity(block, a.log2seq, bytes_per_seq)
    res["fused_step_range"] = {k: [min(v), max(v)] for k, v in res["fused_step_per_s"].items()}
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_r2d2_pool_codec.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
