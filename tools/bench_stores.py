"""The replay store forms of the three learners, measured in one command on one GPU.

    python tools/bench_stores.py --workload apex|r2d2|impala --stores NAME [NAME ...] [--measure NAME [NAME ...]]
        [--batch B [B ...]] [--slots N] [--block N] [--push-batch N] [--steps N] [--warmup N] [--rounds N]
        [--frames random|atari] [--actors N] [--episode E [E]] [--p-done P] [--big-slots N] [--max-host-gb G]
        [--out DIR]

STORES below is the only place that knows the store forms: each is a dict of config overrides on ApexConfig,
R2D2Config or ImpalaConfig.  Records come from the generators under tests/: --frames random gives uniformly random
frames (dedup_model.player_records, strip_dedup_model.player_sequences, impala_rollouts.player_rollouts), --frames
atari the synthetic Atari-like frames of pool_codec_model.atari_frame (apex_atari_records, atari_sequences,
impala_atari_rollouts), both cut as the reference actors cut them, --actors actors interleaved.  No ratio measured on
synthetic frames is a ratio on real Atari frames.  One block of --block records is generated and staged in pinned
buffers of --push-batch records; a store is filled by pushing the block over and over.

Measurements (--measure, default: every one that applies to a chosen store) run over every chosen store they apply to,
the stores alternating, --rounds rounds each:
  bytes     bytes per slot and new frames per record of one pass of the block; for coded stores codec_stats() and the
            b2rl_frame_encode bytes per frame of the distinct frames of the block's first 2048 records (the first
            20 000 in sorted order) and of uniformly random frames
  push      push_arrays records/s from pinned buffers: one pass of the block into a fresh --slots store after one
            warm-up push
  step      the captured in-process fused_step at each --batch over a --slots store, filled, at the library's default
            precision settings (TF32 as torch sets it)
  served    b2rl_serve_fill (IMPALA: b2rl_serve_fill_uniform) into a ring created in this process, and the captured
            bound step (SERVED_FUSED_STEP) on its slots
  capacity  device bytes free before and after creating a --big-slots store, and after filling it past its slot
            ring's wrap (and a coded store's unit ring's, its ring sized from the bytes per record measured first);
            pinned host bytes
  kernels   Ape-X dedup / coded: conv_1's forward of s and of s' and its weight gradient, on the raw pool, decoding in
            conv_1's loader, and decoding into staged stacks first (ms by CUDA events)
  decode    R2D2 coded: GB/s of the decode-assemble gather (k_decode_planes) of a minibatch
  staging   IMPALA coded: b2rl_dedup_stage_rollouts by CUDA events, distinct frames staged per drawn rollout
  host_gather  R2D2 host_pool / host_frames: GB/s of the host-plane and host-row gathers of a minibatch, the
            B2RL_HOST_GATHER_CTAS sweep of the row gather, and the pinned host-to-device cudaMemcpy rate beside it
Prints one JSON line per (measurement, store, batch), each with the card's name, power limit and maximum SM clock; a
figure that is the same in every round is printed once, else one value per round.  Host memory is shared: no store
pins more than --max-host-gb or half of MemAvailable; a store that would is reported as not measured and is never
created.  Pushes and learner steps are timed apart: a push's cost to a learner stepping on the same stream is not
measured.  Needs a GPU; there is no CPU fallback."""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributed_rl_b200 import apex, impala, r2d2, replay as R  # noqa: E402

STORES = {
    "apex": {"stacks": {}, "dedup": {"FRAME_DEDUP": True}, "coded": {"FRAME_DEDUP": True, "FRAME_CODEC": True}},
    "r2d2": {"stacks": {}, "strips": {"FRAME_STRIP": True}, "host_frames": {"FRAME_STRIP": True, "HOST_FRAMES": True},
             "dedup": {"FRAME_DEDUP": True}, "host_pool": {"FRAME_DEDUP": True, "HOST_POOL": True},
             "coded": {"FRAME_DEDUP": True, "POOL_CODEC": True}},
    "impala": {"stacks": {}, "dedup": {"FRAME_DEDUP": True},
               "coded": {"FRAME_DEDUP": True, "STAGED_POOL_CODEC": True}},
}
MODULES = {"apex": apex, "r2d2": r2d2, "impala": impala}
CONFIGS = {"apex": apex.ApexConfig, "r2d2": r2d2.R2D2Config, "impala": impala.ImpalaConfig}
T_R2D2, T_IMPALA = 80, 20        # steps per R2D2 sequence and per IMPALA rollout
BASE = {"apex": {}, "r2d2": {"FIXED_TRAJECTORY": T_R2D2, "MEM": 20}, "impala": {"UNROLL_STEP": T_IMPALA}}
CODED_KEYS = {"apex": ("FRAME_CODEC", "POOL_BYTES_PER_TRANSITION"), "r2d2": ("POOL_CODEC", "POOL_BYTES_PER_SEQUENCE"),
              "impala": ("STAGED_POOL_CODEC", "POOL_BYTES_PER_ROLLOUT")}
FRAMES_PER_SLOT = {"apex": "FRAMES_PER_TRANSITION", "r2d2": "FRAMES_PER_SEQUENCE", "impala": "FRAMES_PER_ROLLOUT"}
DEFAULTS = {   # --batch, --slots, --block, --push-batch, --episode, --big-slots per workload
    "apex": dict(batch=[512], slots=1 << 16, block=16384, push_batch=1024, episode=[400], big_slots=1 << 21),
    "r2d2": dict(batch=[64], slots=1 << 14, block=2048, push_batch=256, episode=[800, 2400], big_slots=1 << 17),
    "impala": dict(batch=[32, 1024], slots=2048, block=2048, push_batch=256, episode=[400, 1600], big_slots=100_000),
}
RING_SLOTS = 4
STRIP_BYTES = (T_R2D2 + 3) * R.FRAME_BYTES       # one R2D2 sequence's frame strip
ROLLOUT_FRAMES = 4 * (T_IMPALA + 1)              # frame positions of one IMPALA rollout's stacks
DISTINCT_RECORDS, DISTINCT_FRAMES = 2048, 20000  # encoded-size sample: distinct frames of the first records
SWEEP = (1, 2, 4, 8, 12, 16, 24, 32, 48, 66, 132)


class NotMeasured(Exception):
    pass


def config(w: str, form: str, slots: int, batch: int = 32, **kw):
    """The learner config of store `form`: the workload's shape, the form's overrides, then `kw`."""
    return CONFIGS[w](**{**BASE[w], **STORES[w][form], "BATCHSIZE": batch, "REPLAY_MEMORY_LEN": slots,
                         "BUFFER_SIZE": 0, "LEARNER_DEVICE": "cuda:0", **kw})


def dedup(w, form) -> bool:
    return bool(STORES[w][form].get("FRAME_DEDUP"))


def coded(w, form) -> bool:
    return bool(STORES[w][form].get(CODED_KEYS[w][0]))


def host_bytes(w, cfg) -> int:
    """Pinned host bytes a store of `cfg` takes: HOST_FRAMES strips or a HOST_POOL frame pool."""
    if getattr(cfg, "HOST_POOL", False):
        return MODULES[w].dedup_geometry(cfg)[0] * R.FRAME_BYTES
    if getattr(cfg, "HOST_FRAMES", False):
        return cfg.REPLAY_MEMORY_LEN * STRIP_BYTES
    return 0


def host_limit(max_host_gb: float) -> int:
    """The most pinned host memory one store may take: --max-host-gb, and half of MemAvailable."""
    with open("/proc/meminfo") as f:
        avail = next(int(line.split()[1]) * 1024 for line in f if line.startswith("MemAvailable"))
    return int(min(max_host_gb * 1e9, avail / 2))


def _checked(w, cfg, args):
    need, limit = host_bytes(w, cfg), host_limit(args.max_host_gb)
    if need > limit:
        raise NotMeasured(f"{need} pinned host bytes needed, above the host limit of {limit} (--max-host-gb, half of "
                          f"MemAvailable)")
    return cfg


def replay(w, form, args, **kw):
    return MODULES[w].Replay(_checked(w, config(w, form, args.slots, **kw), args))


def learner(w, form, args, batch):
    torch.manual_seed(0)
    return MODULES[w].Learner(_checked(w, config(w, form, args.slots, batch), args), start_replay=False)


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


# ---- records and fills ---------------------------------------------------------------------------------------------
_BLOCKS = {}


def records(w, args) -> tuple:
    """The block's records in push_arrays order (priorities not included)."""
    key = ("records", w)
    if key not in _BLOCKS:
        n, atari = args.block, args.frames == "atari"
        if w == "apex":
            if atari:
                from apex_atari_records import atari_records as gen
            else:
                from dedup_model import player_records as gen
            _BLOCKS[key] = gen(n, actors=args.actors, episode=args.episode[0], seed=1)
        elif w == "r2d2":
            if atari:
                from pool_codec_model import atari_sequences as gen
            else:
                from strip_dedup_model import player_sequences as gen
            _BLOCKS[key] = gen(n, T=T_R2D2, actors=args.actors, episode=tuple(args.episode), seed=1)[:6]
        else:
            if atari:
                from impala_atari_rollouts import atari_rollouts as gen
            else:
                from impala_rollouts import player_rollouts as gen
            *recs, kind = gen(n, T=T_IMPALA, actors=args.actors, episode=tuple(args.episode), p_done=args.p_done, seed=1)
            args.padded_rollouts = kind.count("padded")
            _BLOCKS[key] = tuple(recs)
    return _BLOCKS[key]


def chunks(w, form, args) -> list:
    """The block in pinned buffers of --push-batch records, Ape-X and R2D2 priorities last (IMPALA's push takes
    none); an R2D2 stack store gets stacks."""
    stacks = w == "r2d2" and form == "stacks"
    key = ("chunks", w, stacks)
    if key not in _BLOCKS:
        recs = records(w, args)
        if w != "impala":
            recs = (*recs, (np.random.default_rng(2).random(args.block) + 0.05).astype(np.float32))
        out = []
        for i in range(0, args.block, args.push_batch):
            cols = [x[i:i + args.push_batch] for x in recs]
            if stacks:
                cols[0] = cols[0][:, np.arange(T_R2D2)[:, None] + np.arange(4)]
            chunk = []
            for x in cols:
                t = torch.from_numpy(np.ascontiguousarray(x))
                chunk.append(torch.empty(t.shape, dtype=t.dtype, pin_memory=True).copy_(t))
            out.append(chunk)
        _BLOCKS[key] = out
    return _BLOCKS[key]


def fill(memory, block, n) -> float:
    """Push n records (the chunks in `block`, over and over) -> records/s."""
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


def events(fn, n) -> float:
    """ms per call of fn(i), i < n, by CUDA events."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def _finite(out) -> bool:
    return all(bool(torch.isfinite(v).all()) for v in out.values()
               if isinstance(v, torch.Tensor) and v.is_floating_point())


def _close(*stores):
    torch.cuda.synchronize()
    for st in stores:
        st.close()
    gc.collect()
    torch.cuda.empty_cache()


# ---- measurements: generators yielding one round's figures ---------------------------------------------------------
def encoded_bytes(frames: torch.Tensor) -> float:
    """Mean b2rl_frame_encode bytes per frame of (n, 84, 84) uint8 frames."""
    return 16.0 * R.encode_frames(frames.cuda())[1].double().mean().item()


def m_bytes(w, form, args, batch):
    rp = replay(w, form, args)
    ch = chunks(w, form, args)
    fill(rp, ch, args.block)
    st, n = rp.store, args.block
    slot = sum(f.nbytes for f in st.fields)
    out = {"records_pushed": n, "live": len(st), "slot_field_bytes": slot, "bytes_per_slot": slot}
    if dedup(w, form):
        new = st.head_seq / n
        out.update(pool_frames=st.pool_frames, window=st.window, new_frames_per_record=round(new, 3),
                   bytes_per_slot=round(new * R.FRAME_BYTES + slot), bytes_per_slot_at_default_pool=round(
                       getattr(CONFIGS[w], FRAMES_PER_SLOT[w]) * R.FRAME_BYTES + slot))
    if coded(w, form):
        cs = st.codec_stats()
        recs = [x[:DISTINCT_RECORDS] for x in records(w, args)[:2 if w == "apex" else 1]]   # the frame fields
        frames = np.concatenate([x.reshape(len(x), -1) for x in recs], axis=1).reshape(-1, R.FRAME_BYTES)
        distinct = np.unique(frames, axis=0)[:DISTINCT_FRAMES]
        rnd = torch.randint(0, 256, (2048, 84, 84), dtype=torch.uint8, device="cuda",
                            generator=torch.Generator("cuda").manual_seed(5))
        out.update(codec_stats=cs, coded_bytes_per_slot=round(new * cs["bytes_per_frame"] + slot),
                   distinct_frames_encoded=len(distinct),
                   encoded_bytes_per_distinct_frame=round(encoded_bytes(torch.from_numpy(distinct).view(-1, 84, 84)), 1),
                   encoded_bytes_per_random_frame=round(encoded_bytes(rnd), 1))
    _close(st)
    while True:
        yield out


def m_push(w, form, args, batch):
    ch = chunks(w, form, args)
    while True:
        rp = replay(w, form, args)
        rp.push_arrays(*ch[0])                                   # warm-up
        rate = fill(rp, ch[1:], args.block - ch[0][-1].numel())
        _close(rp.store)
        yield {"push_records_per_s": round(rate)}


def m_step(w, form, args, batch):
    L = learner(w, form, args, batch)
    fill(L.memory, chunks(w, form, args), args.slots)
    L.memory.store.seed(7, 0)
    for _ in range(args.warmup):
        L.fused_step(use_graph=True)
    try:
        while True:
            ms = events(lambda i: L.fused_step(use_graph=True), args.steps)
            out = L.fused_step(use_graph=True)
            yield {"steps_per_s": round(1e3 / ms, 1), "live": len(L.memory.store), "steps_finite": _finite(out),
                   "max_idx": int(out["idx"].max())}
    finally:
        _close(L.memory.store)


def ring_fields(w, form):
    return {"apex": lambda: R.APEX_FIELDS, "r2d2": lambda: R.r2d2_fields(T_R2D2, strip=form != "stacks"),
            "impala": lambda: R.impala_fields(T_IMPALA)}[w]()


def m_served(w, form, args, batch):
    from distributed_rl_b200.replay_server import ServeRing
    rp = replay(w, form, args)
    fill(rp, chunks(w, form, args), args.slots)
    st = rp.store
    st.seed(9, 0)
    ring = ServeRing.create(st, batch, RING_SLOTS)
    if w == "impala":
        def serve(k, seed):
            ring.fill_uniform(st, k, seed, T_IMPALA)
    else:
        def serve(k, seed):
            ring.fill(st, k, seed, 0.4)
    for k in range(RING_SLOTS):
        serve(k, k + 1)
    fields = ring_fields(w, form)
    served = {"FRAME_STRIP": form != "stacks"} if w == "r2d2" else {}
    torch.manual_seed(0)
    L = MODULES[w].Learner(CONFIGS[w](**{**BASE[w], **served, "BATCHSIZE": batch, "REPLAY_MEMORY_LEN": 8,
                                         "BUFFER_SIZE": 0, "LEARNER_DEVICE": "cuda:0", "SERVED_FUSED_STEP": True}),
                           start_replay=False, memory=SimpleNamespace(ring=ring, acquire=None, release=None,
                                                                      is_alive=lambda: True))
    s = getattr(L, {"apex": "_fused_state", "r2d2": "_state", "impala": "_bound_state"}[w])()
    bound = (lambda: L.fused_step(use_graph=True)) if w == "apex" else L._bound_step

    def step(i):
        ring.bind(ring.slot_ptrs(i % RING_SLOTS)[0][0], fields, s.cur, s.frames, torch.cuda.current_stream())
        return bound()
    for i in range(args.warmup):
        step(i)
    try:
        while True:
            fill_ms = events(lambda i: serve(i % RING_SLOTS, i + 100), args.steps)
            step_ms = events(step, args.steps)
            yield {"fill_ms": round(fill_ms, 4), "fills_per_s": round(1e3 / fill_ms, 1),
                   "bound_step_per_s": round(1e3 / step_ms, 1), "steps_finite": _finite(step(0))}
    finally:
        torch.cuda.synchronize()
        ring.close()
        _close(st)


def m_capacity(w, form, args, batch):
    n, kw = args.big_slots, {}
    if coded(w, form):
        # the slot ring must wrap before the byte rule evicts: the ring holds the window's raw worst case
        # (7 072 (W + 10) bytes) and 1.25x the coded bytes the block's records added
        rp = replay(w, form, args)
        fill(rp, chunks(w, form, args), args.block)
        per_record = 16.0 * rp.store.codec_stats()["units_written"] / args.block
        _close(rp.store)
        W = MODULES[w].dedup_geometry(config(w, form, n))[1]
        kw[CODED_KEYS[w][1]] = round(1.25 * per_record + 7072 * (W + 10) / n, 1)
    cfg = config(w, form, n, **kw)
    out = {"slots": n, "host_bytes_needed": host_bytes(w, cfg), "host_limit_bytes": host_limit(args.max_host_gb),
           **kw}
    if dedup(w, form):
        F, W = MODULES[w].dedup_geometry(cfg)
        out.update(pool_frames=F, window=W, raw_pool_bytes=F * R.FRAME_BYTES)
    if coded(w, form):
        out["pool_bytes"] = MODULES[w].pool_bytes(cfg)
    try:
        _checked(w, cfg, args)
        need = 0 if dedup(w, form) or host_bytes(w, cfg) else n * sum(f.nbytes for f in ring_fields(w, form))
        if need > torch.cuda.mem_get_info()[0]:
            raise NotMeasured(f"{need} device bytes needed, above the free device memory")
    except NotMeasured as e:
        out.update(measured=False, reason=str(e))
        while True:
            yield out
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    rp = MODULES[w].Replay(cfg)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    pushed = n + n // 2
    rate = fill(rp, chunks(w, form, args), pushed)
    st = rp.store
    out.update(measured=True, device_total=total, device_free_before=free0, device_free_after_create=free1,
               device_free_after_fill=torch.cuda.mem_get_info()[0], store_device_bytes=free0 - free1,
               records_pushed=pushed, live=len(st), fill_records_per_s=round(rate))
    if dedup(w, form):
        out.update(head_seq=st.head_seq, new_frames_per_record=round(st.head_seq / pushed, 3))
        if w == "r2d2":
            out["pool_is_pinned_host"] = bool(st.pool.is_pinned())
    if coded(w, form):
        out["codec_stats"] = st.codec_stats()
    _close(st)
    while True:
        yield out


def m_kernels(w, form, args, batch):
    """conv_1 on the sampled stacks of a filled store: dedup -> raw pool; coded -> decoded in conv_1's loader, and
    decoded into staged stacks by the gather first."""
    rp = replay(w, form, args, batch=batch)
    fill(rp, chunks(w, form, args), args.slots)
    st = rp.store
    g = torch.Generator(device="cuda").manual_seed(3)
    idx = torch.randint(0, len(st), (batch,), device="cuda", generator=g)
    p1, p2 = R.Conv1Pack(1, "cuda"), R.Conv1Pack(2, "cuda")
    wt = torch.randn(32, 4, 8, 8, device="cuda", generator=g) * 0.05
    for p in (p1, p2):
        for k in range(p.n_nets):
            p.pack(k, wt)
    gy = torch.randn(batch, 32, 20, 20, device="cuda", generator=g)
    out1, out2 = torch.empty(1, batch, 20, 20, 32, device="cuda"), torch.empty(2, batch, 20, 20, 32, device="cuda")
    gw = torch.empty(32, 4, 8, 8, device="cuda")
    s, ns = st.frame_source("state"), st.frame_source("next_state")
    arms = {"raw" if form == "dedup" else "in_loader": (
        lambda i: R.conv1_fused(s, idx, p1, relu=True, out=out1), lambda i: R.conv1_fused(ns, idx, p2, relu=False,
                                                                                          out=out2),
        lambda i: R.conv1_wgrad(s, idx, gy, out=gw))}
    extra = {}
    if form == "coded":
        staged = st.alloc_batch(batch, ("state", "next_state"))
        arms["staged"] = (
            lambda i: (st.gather(idx, {"state": staged["state"], "next_state": None}),
                       R.conv1_fused(staged["state"], None, p1, relu=True, out=out1)),
            lambda i: (st.gather(idx, {"next_state": staged["next_state"], "state": None}),
                       R.conv1_fused(staged["next_state"], None, p2, relu=False, out=out2)),
            lambda i: R.conv1_wgrad(staged["state"], None, gy, out=gw))
        y_in = R.conv1_fused(ns, idx, p2)
        st.gather(idx, {"next_state": staged["next_state"], "state": None})
        extra["in_loader_equals_staged"] = all(torch.equal(u, v) for u, v in zip(y_in, R.conv1_fused(
            staged["next_state"], None, p2)))
    for fns in arms.values():
        for fn in fns:
            events(fn, 5)
    try:
        while True:
            yield {**{f"{arm}_ms_fwd_s_fwd_ns_wgrad": [round(events(fn, args.steps), 4) for fn in fns]
                      for arm, fns in arms.items()}, **extra}
    finally:
        _close(st)


def _gather_gbps(st, idx, out, iters) -> float:
    for _ in range(5):
        st.gather(idx, out)
    return round(idx.numel() * STRIP_BYTES / (events(lambda i: st.gather(idx, out), iters) / 1e3) / 1e9, 2)


def m_decode(w, form, args, batch):
    rp = replay(w, form, args)
    fill(rp, chunks(w, form, args), args.slots)
    st = rp.store
    idx = torch.randint(0, len(st), (batch,), device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    out = st.alloc_batch(batch, ("state",))
    try:
        while True:
            yield {"decode_GBps": _gather_gbps(st, idx, out, args.steps), "minibatch_bytes": batch * STRIP_BYTES}
    finally:
        _close(st)


def m_staging(w, form, args, batch):
    rp = replay(w, form, args)
    fill(rp, chunks(w, form, args), args.slots)
    st = rp.store
    cur = {"idx": torch.empty(batch, dtype=torch.int64, device="cuda")}
    st.seed(5, 0)
    st.uniform_fetch(batch, T_IMPALA, cur)
    staged = st.alloc_staged(batch)
    st.stage_frames(cur["idx"], staged)
    first = staged["planes"] == torch.arange(batch * ROLLOUT_FRAMES, device="cuda", dtype=torch.int32).view(batch, ROLLOUT_FRAMES)
    distinct = first.sum().item() / batch
    try:
        while True:
            ms = events(lambda i: st.stage_frames(cur["idx"], staged), args.steps)
            yield {"distinct_frames_per_rollout": round(distinct, 2), "stage_us": round(1e3 * ms, 1),
                   "staged_frames_per_s": round(distinct * batch / ms * 1e3)}
    finally:
        del staged
        _close(st)


def memcpy_gbps(nbytes: int, iters: int = 50) -> float:
    """Pinned host -> device cudaMemcpy GB/s of one nbytes buffer."""
    from distributed_rl_b200 import hostmem
    h = hostmem.pinned_empty((nbytes,), torch.uint8, "cuda:0")
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(10):
            d.copy_(h, non_blocking=True)
        ms = events(lambda i: d.copy_(h, non_blocking=True), iters)
    return round(nbytes / (ms / 1e3) / 1e9, 2)


def m_host_gather(w, form, args, batch):
    """host_pool: k_gather_host_planes (strips of scattered pool frames); host_frames: k_gather_host_rows
    (contiguous strips) at the default CTA count and over the B2RL_HOST_GATHER_CTAS sweep."""
    rp = replay(w, form, args)
    fill(rp, chunks(w, form, args), args.slots)
    st = rp.store
    idx = torch.randint(0, len(st), (batch,), device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    out = st.alloc_batch(batch, ("state",))
    try:
        while True:
            res = {"gather_GBps": _gather_gbps(st, idx, out, args.steps), "minibatch_bytes": batch * STRIP_BYTES,
                   "memcpy_h2d_GBps": memcpy_gbps(batch * STRIP_BYTES)}
            if form == "host_frames":
                saved = os.environ.get("B2RL_HOST_GATHER_CTAS")
                try:
                    res["GBps_by_ctas"] = {}
                    for ctas in SWEEP:
                        os.environ["B2RL_HOST_GATHER_CTAS"] = str(ctas)
                        res["GBps_by_ctas"][ctas] = _gather_gbps(st, idx, out, args.steps)
                finally:
                    os.environ.pop("B2RL_HOST_GATHER_CTAS")
                    if saved is not None:
                        os.environ["B2RL_HOST_GATHER_CTAS"] = saved
                res["last_gather_matches_index_select"] = torch.equal(
                    out["state"].cpu(), st.field_view("state").index_select(0, idx.cpu()))
            yield res
    finally:
        _close(st)


# name -> (function, stores it applies to (None: all), runs at each --batch)
MEASURES = {
    "bytes": (m_bytes, None, False),
    "push": (m_push, None, False),
    "step": (m_step, None, True),
    "served": (m_served, None, True),
    "capacity": (m_capacity, None, False),
    "kernels": (m_kernels, {"apex": ("dedup", "coded")}, True),
    "decode": (m_decode, {"r2d2": ("coded",)}, True),
    "staging": (m_staging, {"impala": ("coded",)}, True),
    "host_gather": (m_host_gather, {"r2d2": ("host_pool", "host_frames")}, True),
}
ONCE = ("bytes", "capacity")           # the same in every round: measured once


def applies(name, w, form) -> bool:
    only = MEASURES[name][1]
    return only is None or form in only.get(w, ())


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workload", required=True, choices=sorted(STORES))
    ap.add_argument("--stores", nargs="+", required=True, help="store forms: " + "; ".join(
        f"{w}: {' '.join(STORES[w])}" for w in STORES))
    ap.add_argument("--measure", nargs="+", choices=list(MEASURES), help="default: every one that applies")
    ap.add_argument("--batch", type=int, nargs="+")
    ap.add_argument("--slots", type=int, help="slots of the stores pushed, stepped and served")
    ap.add_argument("--block", type=int, help="records generated and staged in pinned buffers")
    ap.add_argument("--push-batch", type=int)
    ap.add_argument("--steps", type=int, default=100, help="timed calls per round")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", choices=("random", "atari"), default="random")
    ap.add_argument("--actors", type=int, default=32)
    ap.add_argument("--episode", type=int, nargs="+", help="Ape-X: frames per episode; R2D2, IMPALA: min max steps")
    ap.add_argument("--p-done", type=float, default=0.01, help="IMPALA: a life lost per step")
    ap.add_argument("--big-slots", type=int, help="slots of the capacity store")
    ap.add_argument("--max-host-gb", type=float, default=16.0)
    ap.add_argument("--out", help="also write the JSON lines to DIR/bench_stores.jsonl")
    a = ap.parse_args(argv)
    for k, v in DEFAULTS[a.workload].items():
        if getattr(a, k) is None:
            setattr(a, k, v)
    unknown = [s for s in a.stores if s not in STORES[a.workload]]
    if unknown:
        ap.error(f"unknown {a.workload} store {' '.join(unknown)}: choose from {' '.join(STORES[a.workload])}")
    for name in a.measure or ():
        if not any(applies(name, a.workload, s) for s in a.stores):
            ap.error(f"--measure {name} does not apply to {a.workload} {' '.join(a.stores)}")
    a.measure = a.measure or [m for m in MEASURES if any(applies(m, a.workload, s) for s in a.stores)]
    a.configs = {s: config(a.workload, s, a.slots, a.batch[0]) for s in a.stores}   # the configs' own checks
    return a


def _merge(rounds: list) -> dict:
    """One round's figures -> the figure; several -> one value per round, or one value if all rounds agree."""
    return {k: (rounds[0][k] if all(r[k] == rounds[0][k] for r in rounds) else [r[k] for r in rounds])
            for k in rounds[0]}


def main(argv=None):
    a = parse(argv)
    if not torch.cuda.is_available():
        sys.exit("bench_stores measures the stores on the GPU: needs a GPU")
    head = {"card": card(), "workload": a.workload, "frames": a.frames}
    sink = None
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        sink = open(os.path.join(a.out, "bench_stores.jsonl"), "a")
    for name in a.measure:
        fn, _, batched = MEASURES[name]
        forms = [s for s in a.stores if applies(name, a.workload, s)]
        for batch in (a.batch if batched else [None]):
            gens, res = {}, {s: [] for s in forms}
            try:
                for s in forms:
                    gens[s] = fn(a.workload, s, a, batch or a.batch[0])
                for r in range(1 if name in ONCE else a.rounds):
                    for s in (forms if r % 2 == 0 else forms[::-1]):
                        if s in gens:
                            try:
                                res[s].append(next(gens[s]))
                            except NotMeasured as e:
                                res[s] = [{"measured": False, "reason": str(e)}]
                                del gens[s]
            finally:
                for g in gens.values():
                    g.close()
            for s in forms:
                line = dict(head, measure=name, store=s, batch=batch, **_merge(res[s]))
                if name in ("bytes", "push") and a.workload == "impala":
                    line["padded_rollouts"] = getattr(a, "padded_rollouts", None)
                print(json.dumps(line), flush=True)
                if sink:
                    sink.write(json.dumps(line) + "\n")
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
