"""Stand-alone replay server transports, Ape-X transitions, R2D2 sequences or IMPALA rollouts at batch B: served
minibatches/s and learner steps/s for
  redis   ReplayServer -> pickled `BATCH` list -> Replay_Server (host arrays, copied to the device by train());
          Ape-X and R2D2 only
  ring    DeviceReplayServer -> device serve ring (CUDA IPC) -> DeviceReplayClient
  ring-fused  the same ring, with the learner's captured step reading each minibatch in its ring slot
          (SERVED_FUSED_STEP: acquire -> graph replay -> release -> write-back, IMPALA without the write-back);
          served minibatches/s is acquire + release alone
  fused   the in-process learner: Learner.fused_step() on its own replay (no server); captured for Ape-X, eager for
          R2D2 and IMPALA
  fused-graph  R2D2 and IMPALA: the in-process fused_step(use_graph=True), captured in its first call and replayed
          (IMPALA: one b2rl_uniform_fetch draw launch before each replay)
  sample  IMPALA only: the in-process Replay's sample() -> Learner.train() (gather + time-major transpose per step)
  fill    b2rl_serve_fill (IMPALA: b2rl_serve_fill_uniform) alone, in this process: CUDA events around `steps` fills
          into alternating ring slots, at each batch of --fill-batches; bytes/s = 2 x slot bytes / fill time (each
          byte read once, written once)

    python tools/bench_serve.py [--workload apex|r2d2|impala] [--slots-store N] [--batch B] [--steps 200]
                                [--warmup 20] [--repeats 3]
                                [--arms redis,ring,ring-fused,fused,fused-graph,sample,fill]

Defaults per workload: Ape-X B = 512 on a 2^16-slot store (3.7 GB); R2D2 B = 64, T = 80, MEM = 20 on a 2^12-sequence
store (9.2 GB); IMPALA B = 32, T = 20 on a 2^11-rollout store (1.2 GB).

The server runs in a `spawn` child on --server-device, the learner here on cuda:0; the control plane is a Redis
server (--redis HOST) or, by default, the in-memory Redis stand-in of the tests hosted by a multiprocessing manager
(tests/shared_redis.py).  The stand-in moves the Redis-pickle arm's 29 MB minibatches through a Python socket and is
much slower than a Redis server: that arm is then a lower bound, not a representative baseline.  With both processes on ONE GPU
they share its SMs, so the served figures are a lower bound for a server with a GPU of its own.  Timings: host
clock around `steps` iterations that end in a device synchronise, after `warmup` iterations; every arm is repeated
`repeats` times in alternation and each run is reported.  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import multiprocessing as mp
import os
import pickle
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from shared_redis import RedisManager, Shim  # noqa: E402


def _connect(args, proxy):
    """The control plane: a Redis server when --redis HOST is given, else the manager-hosted stand-in."""
    if args["redis"]:
        import redis
        return redis.StrictRedis(host=args["redis"], port=6379)
    return Shim(proxy)


def _cfg(args, device):
    from distributed_rl_b200 import apex, impala, r2d2
    if args["workload"] == "impala":
        return impala.ImpalaConfig(BATCHSIZE=args["batch"], UNROLL_STEP=20, REPLAY_MEMORY_LEN=args["store"],
                                   BUFFER_SIZE=0, LEARNER_DEVICE=device)
    if args["workload"] == "r2d2":
        return r2d2.R2D2Config(BATCHSIZE=args["batch"], REPLAY_MEMORY_LEN=args["store"], BUFFER_SIZE=0,
                               FIXED_TRAJECTORY=80, MEM=20, LEARNER_DEVICE=device)
    return apex.ApexConfig(BATCHSIZE=args["batch"], REPLAY_MEMORY_LEN=args["store"], BUFFER_SIZE=0,
                           LEARNER_DEVICE=device)


def _learner(args, cfg, memory=None):
    from distributed_rl_b200 import apex, impala, r2d2
    mod = {"r2d2": r2d2, "impala": impala}.get(args["workload"], apex)
    return mod.Learner(cfg, connect=None, start_replay=False, **({} if memory is None else {"memory": memory}))


def _fill(store, n):
    import torch
    store.fill_hash(n, seed=0xB200)
    store.build(torch.rand(n, generator=torch.Generator().manual_seed(0)).to(store.device) + 1e-3)
    if "mu" in [f.name for f in store.fields]:
        # IMPALA rollouts: Learner.train indexes the policy with the stored actions, so hashed words will not do
        g = torch.Generator(device=store.device).manual_seed(0)
        store.field_view("action").random_(0, 6, generator=g)          # ImpalaConfig.ACTION_SIZE
        store.field_view("mu").uniform_(0.1, 1.0, generator=g)
        store.field_view("reward").normal_(generator=g)
        store.field_view("done").bernoulli_(0.9, generator=g)


def _server_main(kind, proxy, args, stop):
    """Serve until `stop`: the ring server keeps its slots full; the Redis server keeps <= 8 pickled batches queued."""
    from distributed_rl_b200.replay_server import DeviceReplayServer, ReplayServer
    conn = _connect(args, proxy)
    cfg = _cfg(args, args["server_device"])
    if kind.startswith("ring"):
        srv = DeviceReplayServer(cfg, conn, slots=args["ring_slots"])
        _fill(srv.store, args["store"])
        while not stop.is_set():
            st = srv.serve_once()
            if not (st["filled"] or st["released"] or st["updates_applied"]):
                time.sleep(0.0002)
        srv.close()
    else:
        srv = ReplayServer(cfg, conn, conn, m=1)
        _fill(srv.store, args["store"])
        conn.set("SERVE_STATS", pickle.dumps((args["store"], 1.0)))
        while not stop.is_set():
            busy = srv.update()
            if conn.llen("BATCH") < 8:
                srv.buffer()
                busy = True
            if not busy:
                time.sleep(0.0002)


def _timed(fn, steps, warmup, dev):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize(dev)
    return steps / (time.perf_counter() - t0)


def _served_arm(kind, args):
    import torch
    from distributed_rl_b200.replay_server import DeviceReplayClient, Replay_Server
    ctx = mp.get_context("spawn")
    mgr = RedisManager(ctx=ctx)
    mgr.start()
    stop, child, client = ctx.Event(), None, None
    dev = torch.device("cuda:0")
    try:
        proxy = mgr.Redis()
        conn = _connect(args, proxy)
        child = ctx.Process(target=_server_main, args=(kind, proxy, args, stop))
        child.start()
        cfg = _cfg(args, "cuda:0")
        cfg.CUDNN_BENCHMARK = True
        cfg.SERVED_FUSED_STEP = kind == "ring-fused"
        if kind.startswith("ring"):
            client = DeviceReplayClient(cfg, conn, timeout=300.0)
        else:
            client = Replay_Server(cfg, conn, conn)
            client.start()
        L = _learner(args, cfg, client)
        frames = (1,) if args["workload"] == "r2d2" else (0, 3)     # the frame arrays of the minibatch list

        def next_batch():
            while (b := client.sample()) is False:
                time.sleep(0.0001)
            return b

        def serve_only():
            b = next_batch()
            if kind == "redis":          # what train() would do first: the batch onto the device
                for i in frames:
                    b[i] = torch.as_tensor(b[i]).to(dev, non_blocking=True)

        def step():
            b = next_batch()
            if args["workload"] == "impala":        # uniform replay: no priorities to write back
                L.train(b)
                return
            info, prio, idx = L.train(b)[:3]
            client.update(idx if kind == "ring" else list(idx.tolist()), prio)
        if kind == "ring-fused":
            s = getattr(L, {"r2d2": "_state", "impala": "_bound_state"}.get(args["workload"], "_fused_state"))()
            count = [0]

            def serve_only():            # the bind alone: acquire (wait on filled[k] + one k_serve_bind), release
                while client.acquire(s.cur, s.frames) is None:
                    time.sleep(0.0001)
                client.release()

            def step():                  # the eviction request never comes: every step writes back (not IMPALA)
                count[0] += 1
                if args["workload"] == "impala":
                    while not L._next_step(count[0]):
                        time.sleep(0.0001)
                    return
                while L._next_step(count[0], 1 << 62) is None:
                    time.sleep(0.0001)
        n = args["redis_steps"] if kind == "redis" else args["steps"]
        served = _timed(serve_only, n, args["warmup"], dev)
        steps = _timed(step, n, args["warmup"], dev)
        return {"served_minibatches_per_s": served, "learner_steps_per_s": steps}
    finally:
        stop.set()
        if client is not None:
            client.stop()
            if kind.startswith("ring"):
                client.close()
            else:
                client.join(timeout=10)        # the polling thread must not outlive the manager
        if child is not None:
            child.join(timeout=60)
            if child.is_alive():
                child.terminate()
                child.join()
        mgr.shutdown()


def _fused_arm(args, use_graph=False):
    """The in-process fused_step: eager (`fused`) or, R2D2's and IMPALA's `fused-graph`, captured in the first call
    and replayed (the warm-up calls include the three eager warm-ups and the capture)."""
    import torch
    cfg = _cfg(args, "cuda:0")
    L = _learner(args, cfg)
    _fill(L.memory.store, args["store"])
    fn = (lambda: L.fused_step(use_graph=True)) if use_graph else L.fused_step
    rate = _timed(fn, args["steps"], args["warmup"], torch.device("cuda:0"))
    del L
    torch.cuda.empty_cache()
    return {"served_minibatches_per_s": None, "learner_steps_per_s": rate}


def _sample_arm(args):
    """IMPALA's in-process path through the learner's own replay: Replay.sample() (draw, gather, transpose to
    time-major) -> Learner.train()."""
    import torch
    cfg = _cfg(args, "cuda:0")
    L = _learner(args, cfg)
    _fill(L.memory.store, args["store"])
    rate = _timed(lambda: L.train(L.memory.sample()), args["steps"], args["warmup"], torch.device("cuda:0"))
    del L
    torch.cuda.empty_cache()
    return {"served_minibatches_per_s": None, "learner_steps_per_s": rate}


def _fill_arm(args):
    """b2rl_serve_fill alone: one store, a 2-slot ring per batch size, CUDA events around `steps` back-to-back
    fills (slots alternate, as a server with a free slot would fill them)."""
    import torch
    from distributed_rl_b200 import replay as R
    from distributed_rl_b200.replay_server import ServeRing, record_kind
    cfg = _cfg(args, "cuda:0")
    kind = record_kind(cfg)
    store = R.DeviceReplay(args["store"], kind.fields(cfg), "cuda:0")
    _fill(store, args["store"])
    out = {}
    try:
        for B in args["fill_batches"]:
            ring = ServeRing.create(store, B, 2)

            def fill(i):
                if kind.prioritized:
                    ring.fill(store, i % 2, i + 1, cfg.BETA)
                else:
                    ring.fill_uniform(store, i % 2, i + 1, kind.steps(cfg))
            for i in range(args["warmup"]):
                fill(i)
            st = torch.cuda.current_stream()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for i in range(args["steps"]):
                fill(i)
            e1.record(st)
            e1.synchronize()
            t = e0.elapsed_time(e1) / 1e3 / args["steps"]
            bps = 2 * ring.layout.slot_bytes / t
            out[str(B)] = {"fill_us": t * 1e6, "slot_bytes": ring.layout.slot_bytes, "bytes_per_s": bps,
                           "fraction_of_3.35e12": bps / 3.35e12}
            torch.cuda.synchronize()
            ring.close()
    finally:
        store.close()
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("apex", "r2d2", "impala"), default="apex")
    ap.add_argument("--slots-store", type=int, default=None,
                    help="replay slots (default: Ape-X 2^16 = 3.7 GB, R2D2 2^12 sequences = 9.2 GB, IMPALA 2^11 "
                         "rollouts = 1.2 GB)")
    ap.add_argument("--batch", type=int, default=None, help="default: Ape-X 512, R2D2 64, IMPALA 32")
    ap.add_argument("--fill-batches", default=None, help="batch sizes of the fill arm, e.g. 32,64 (default: --batch)")
    ap.add_argument("--redis-steps", type=int, default=None, help="timed steps of the redis arm (default: --steps)")
    ap.add_argument("--ring-slots", type=int, default=4)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--server-device", default="cuda:0")
    ap.add_argument("--arms", default=None, help="any of redis, ring, ring-fused, fused, fused-graph (R2D2, IMPALA), "
                    "sample, "
                    "fill (default: Ape-X and R2D2 redis,ring,fused; IMPALA ring,sample,fused)")
    ap.add_argument("--redis", default=None, help="host of a Redis server for the control plane (default: an "
                    "in-memory stand-in in a manager process, which makes the Redis-pickle arm far slower than a "
                    "Redis server would)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_serve.py measures on a CUDA device; none is available")
    store = a.slots_store or {"r2d2": 4096, "impala": 2048}.get(a.workload, 65536)
    batch = a.batch or {"r2d2": 64, "impala": 32}.get(a.workload, 512)
    arms = a.arms or ("ring,sample,fused" if a.workload == "impala" else "redis,ring,fused")
    if a.workload == "impala" and "redis" in arms.split(","):
        sys.exit("IMPALA has no Redis-protocol replay server")
    if a.workload == "apex" and "fused-graph" in arms.split(","):
        sys.exit("the fused-graph arm is the R2D2 and IMPALA learners' captured in-process step (Ape-X's fused arm is "
                 "captured already)")
    args = {"workload": a.workload, "store": store, "batch": batch, "ring_slots": a.ring_slots, "steps": a.steps,
            "warmup": a.warmup, "server_device": a.server_device, "redis": a.redis,
            "redis_steps": a.redis_steps or a.steps,
            "fill_batches": [int(x) for x in a.fill_batches.split(",")] if a.fill_batches else [batch]}
    runs = {k: [] for k in arms.split(",")}
    arm = {"fused": _fused_arm, "fused-graph": lambda x: _fused_arm(x, use_graph=True), "sample": _sample_arm,
           "fill": _fill_arm}
    for _ in range(a.repeats):
        for k in runs:
            runs[k].append(arm[k](args) if k in arm else _served_arm(k, args))
            print(json.dumps({"arm": k, **runs[k][-1]}), file=sys.stderr, flush=True)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    except Exception:
        q = []
    same = a.server_device == "cuda:0"
    print(json.dumps({"workload": f"{a.workload}_serve", "batch": batch, "store_slots": store,
                      "server_device": a.server_device, "learner_device": "cuda:0",
                      "control_plane": f"redis://{a.redis}" if a.redis else "in-memory stand-in (manager process)",
                      "note": "server and learner share one GPU: served figures are a lower bound" if same else
                      "server and learner on separate GPUs",
                      "gpus": q, "runs": runs}))


if __name__ == "__main__":
    main()
