"""What the Ape-X, R2D2 and IMPALA learner sides share: the optimiser factory, the replay ingest thread and the
learner's replay set-up, the conv_1 autograd function and its packs, the time-major frame-row layout, the checks
and the warm-up / capture / replay of a captured step (`CapturedStep`), and the Ape-X / R2D2 `Learner.run` loop with
its write-back cadence (start handshake, publishers, periodic log).  Each learner keeps its own store layout, batch
assembly and step body."""
from __future__ import annotations

import pickle
import threading
import time

import numpy as np
import torch

from . import _lib
from . import replay as R
from . import wire
from .publish import ParamPublisher


def make_optimizer(info: dict, params, capturable: bool = True):
    """baseline/utils.py getOptim (:78-132) for the optimisers the shipped configs name."""
    name = info["name"]
    lr, decay, eps = info["lr"], info.get("decay", 0), info.get("eps", 1e-5)
    if name == "rmsprop":
        return torch.optim.RMSprop(params, lr=lr, weight_decay=decay, eps=eps, momentum=info.get("momentum", 0),
                                   alpha=info.get("alpha", 0.99), centered=info.get("centered", False),
                                   capturable=capturable, foreach=True)
    if name == "adam":
        return torch.optim.Adam(params, lr=lr, weight_decay=decay, eps=eps,
                                betas=(info.get("beta1", 0.9), info.get("beta2", 0.99)),
                                capturable=capturable, foreach=True)
    if name == "sgd":
        return torch.optim.SGD(params, lr=lr, weight_decay=decay, momentum=info.get("momentum", 0))
    raise ValueError(f"unknown optimizer {name!r}")


class MemoryView:
    """What the learner reads from `Replay.memory` (APE_X/Learner.py:143,241):
    len() and .max_weight (baseline/PER.py:80-81,129-133)."""

    def __init__(self, dev_replay: R.DeviceReplay, beta: float):
        self._r, self._beta = dev_replay, beta

    def __len__(self):
        return len(self._r)

    @property
    def max_weight(self) -> float:
        return float(self._r.stats(self._beta)[2].item())


# -- replay ingest threads ------------------------------------------------------------------------
class Stoppable:
    """`stop()` for a polling loop (the reference's daemon threads can only die with the process).  The event is
    `_stop_evt`, NOT `_stop`: that name is threading.Thread's own method."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._stop_evt = threading.Event()

    def stop(self) -> None:
        """Ask the loop to leave."""
        self._stop_evt.set()


class ReplayThread(Stoppable, threading.Thread):
    """The `Replay` thread of APE_X/ReplayMemory.py (:19-167), R2D2/ReplayMemory.py and IMPALA/ReplayMemory.py.
    A subclass sets `self.store` (the DeviceReplay the sum-tree lives in) and provides `push_records(blobs)` and
    `buffer(m)`, which appends m assembled minibatches to `deque`."""

    LIST_KEY = "experience"     # the actors' Redis list drained by run()

    def __init__(self, cfg, connect=None):
        super().__init__(daemon=True)
        self.cfg = cfg
        self.device = torch.device(cfg.LEARNER_DEVICE)
        self.connect = connect
        self.cond = False
        self.lock = False          # eviction request from the learner, served by run()
        self.deque = []            # pre-assembled minibatches (filled on demand)
        self.total_frame = 0
        self._lock = threading.Lock()

    def run(self):
        """Poll the actors' Redis list like APE_X/ReplayMemory.py:118-161: drain `LIST_KEY`, push, honour the
        learner's eviction request (`lock`, :151-160).  Minibatches are assembled on demand by sample()."""
        if self.connect is None:
            return
        while not self._stop_evt.is_set():
            data = wire.drain(self.connect, self.LIST_KEY)
            if data:
                self.push_records(data)
                self.cond = len(self.store) > self.cfg.BUFFER_SIZE
            if self.lock:
                self._evict_on_request()
            if not data:
                time.sleep(0.002)

    def _wire_decode(self, blobs):
        """push_records' device path: the pickled records decoded on the GPU by the subclass's wire.WireIngest (made on
        first use), or None for the host path: a replay not on a GPU, or a batch the device path hands back whole."""
        if torch.device(self.cfg.LEARNER_DEVICE).type != "cuda":
            return None
        if self.__dict__.get("_wire") is None:
            self._wire = self._wire_ingest()
        return self._wire.decode(blobs)

    def _evict_on_request(self) -> None:
        """The `lock` handshake (APE_X/ReplayMemory.py:151-160, APE_X/Learner.py:189-197): once the memory is full,
        drop queued minibatches and trim to REPLAY_MEMORY_LEN (PER.remove_to_fit, baseline/PER.py:118-127).  The
        ring already overwrites its oldest slot on push, so there is normally nothing to trim."""
        if len(self.store) >= self.cfg.REPLAY_MEMORY_LEN:
            with self._lock:
                self.deque.clear()
                over = len(self.store) - self.cfg.REPLAY_MEMORY_LEN
                if over > 0:
                    self.store.evict(over)
        self.lock = False

    def sample(self):
        """The next queued minibatch, assembling one if none is queued; False until more than BUFFER_SIZE records
        are stored."""
        if not self.deque:
            if len(self.store) <= self.cfg.BUFFER_SIZE:
                return False
            self.buffer(1)
        return self.deque.pop(0)

    def update(self, idx, vals) -> None:
        """Replay.update (APE_X/ReplayMemory.py:43-59) -> PER.update, applied at once.  `idx`: see _index_tensor."""
        with self._lock:
            self.store.update(_index_tensor(idx).to(self.device), torch.as_tensor(vals).to(self.device))


def _index_tensor(idx) -> torch.Tensor:
    """A write-back's replay slots as a tensor.  `idx`: a tensor, an array, or a list of ints or 0-d tensors (what
    the reference passes)."""
    if isinstance(idx, (list, tuple)):
        return torch.stack([torch.as_tensor(i) for i in idx]) if len(idx) and torch.is_tensor(idx[0]) \
            else torch.as_tensor(np.asarray(idx, np.int64))
    return torch.as_tensor(idx)


def _attach_replay(learner, memory, make_replay, connect, start_replay: bool, wipe: bool):
    """The learner's replay (APE_X/Learner.py:28-29,41-43, R2D2/Learner.py:46-48,54,63-64, IMPALA/Learner.py:27-28):
    `memory`, a replay served from another process, started unless it already runs; or, when it is None,
    `make_replay()`, the learner's own, started when there is a Redis connection.  `wipe`: then drop whatever a
    previous run left in the database, except the keys of a replay server this learner is attached to
    (`memory.KEEP_KEYS`: its handshake lives there).  Sets `learner._served`.  -> the replay."""
    learner._served = memory is not None
    if learner._served:
        if start_replay and not memory.is_alive():
            memory.start()
    else:
        memory = make_replay()
        if start_replay and connect is not None:
            memory.start()
    if wipe and connect is not None:
        wire.wipe_stale_keys(connect, keep=getattr(memory, "KEEP_KEYS", ()) if learner._served else ())
    return memory


# -- conv_1 on libb2rl's kernels -----------------------------------------------------------------
class Conv1Gathered(torch.autograd.Function):
    """conv_1 over rows `idx` of a uint8 frame table (a replay field, an explicit batch, or a served ring slot bound
    through a device-resident table entry, R.BoundFrames: backward then reads the same slot rows).
    Forward: fused gather+conv on the tensor cores (or a precomputed output of the same kernel).
    Backward: only dL/dW is needed (the input is data); cuDNN computes it from a gathered fp32
    copy of the same rows — the one place the sampled frames are staged — or, with `fused_wgrad`
    (default), libb2rl's fused gather + wgrad kernel computes it from the uint8 rows directly."""

    fused_wgrad = True

    @staticmethod
    def forward(ctx, weight, frames, idx, pack, mem_format, store=None, y_pre=None, relu=False):
        """relu=True: the kernel's epilogue applies the ReLU that follows conv_1 and backward applies its mask
        inside the wgrad kernel (the caller must then skip the network's own ReLU: forward_from_conv1(y, True))."""
        ctx.frames, ctx.store, ctx.mem_format, ctx.wshape = frames, store, mem_format, weight.shape
        ctx.weight_param = weight
        ctx.has_idx, ctx.relu = idx is not None, bool(relu)
        idx_t = idx if idx is not None else torch.empty(0, dtype=torch.int64, device=frames.device)
        if y_pre is not None:
            y = y_pre.view_as(y_pre)
        else:
            y = R.conv1_fused(frames, idx, pack, relu=bool(relu))[0]
        if relu:
            ctx.save_for_backward(idx_t, y)
        else:
            ctx.save_for_backward(idx_t)
        return y

    @staticmethod
    def backward(ctx, gy):
        idx = ctx.saved_tensors[0]
        y = ctx.saved_tensors[1] if ctx.relu else None
        if Conv1Gathered.fused_wgrad:
            # fused gather + wgrad on the tensor cores: the sampled rows are never staged (csrc/conv1_wgrad.cu)
            w = ctx.weight_param
            from . import linear as _lin
            if _lin._SINK is not None and w.grad is not None and w.grad.is_contiguous():
                # deferred-gradient mode (grads pre-allocated, zeroed by the optimizer): the kernel's reduction adds
                # straight into .grad — no temporary, no AccumulateGrad launch at the very end of backward
                R.conv1_wgrad(ctx.frames, idx if ctx.has_idx else None, gy, out=w.grad, accumulate=True, relu_y=y)
                return (None,) * len(ctx.needs_input_grad)
            gw = R.conv1_wgrad(ctx.frames, idx if ctx.has_idx else None, gy, relu_y=y)
            return (gw,) + (None,) * (len(ctx.needs_input_grad) - 1)
        if isinstance(ctx.frames, (R.BoundFrames, R.PlaneFrames, R.CodedPlaneFrames)):
            raise RuntimeError("conv_1 over a bound ring slot or a frame pool has no cuDNN weight gradient: set "
                               "Conv1Gathered.fused_wgrad")
        if y is not None:
            gy = gy * (y > 0)
        if not ctx.has_idx:
            x = ctx.frames
        elif ctx.store is not None and ctx.frames.stride(0) == R.FRAME_STACK_BYTES:
            # TMA bulk gather straight from the replay payload (whole records: never for the windows of frame strips)
            x = ctx.store.gather(idx, ctx.store.alloc_batch(idx.numel(), ("state",)))["state"]
        else:
            x = ctx.frames.index_select(0, idx)
        xf = (x.to(torch.float32) / 255.0).contiguous(memory_format=ctx.mem_format)
        gw = torch.nn.grad.conv2d_weight(xf, ctx.wshape, gy.contiguous(memory_format=ctx.mem_format), stride=4)
        return (gw,) + (None,) * (len(ctx.needs_input_grad) - 1)


class StemGathered(torch.autograd.Function):
    """The residual network's stem (3x3 conv + max-pool, R.stem_fused) over rows `idx` of a uint8 frame table, as
    Conv1Gathered is conv_1: forward returns the pooled output the fused kernel already computed (`pooled`, with its
    `argmax`); backward computes only dL/dW (the input is data) with the fused weight-gradient kernel, the max-pool's
    backward folded into its loader through `argmax`, from the same rows read in place."""

    @staticmethod
    def forward(ctx, weight, frames, idx, pooled, argmax):
        ctx.frames, ctx.weight_param, ctx.has_idx = frames, weight, idx is not None
        idx_t = idx if idx is not None else torch.empty(0, dtype=torch.int64, device=frames.device)
        ctx.save_for_backward(idx_t, argmax)
        return pooled.view_as(pooled)

    @staticmethod
    def backward(ctx, gp):
        idx, argmax = ctx.saved_tensors
        idx = idx if ctx.has_idx else None
        w = ctx.weight_param
        from . import linear as _lin
        if _lin._SINK is not None and w.grad is not None and w.grad.is_contiguous():
            R.stem_wgrad(ctx.frames, idx, gp, argmax, out=w.grad, accumulate=True)
            return (None,) * len(ctx.needs_input_grad)
        return (R.stem_wgrad(ctx.frames, idx, gp, argmax),) + (None,) * (len(ctx.needs_input_grad) - 1)


def fused_first_layer(model) -> bool:
    """True if the model's first layer reads frames on libb2rl's kernels: the Atari conv_1, or the stem of a RESCNN2D
    node (GraphAgent.first_stem_node)."""
    return model.first_conv_node() is not None or model.first_stem_node() is not None


def require_fused_first_layer(model, what: str) -> None:
    """ValueError naming `what` (the step that reads the frames in place) unless fused_first_layer(model)."""
    if not fused_first_layer(model):
        raise ValueError(f"{what} reads the frames with the fused conv_1 or stem kernels: the model's first node must be "
                         "the Atari conv_1 or a RESCNN2D stem")


def conv1_packs(model, device, *n_nets):
    """-> (name of `model`'s first conv node, one Conv1Pack per entry of `n_nets`): each pack holds the conv_1
    weights of that many networks (1: online; 2: online + target, run as one launch)."""
    name = model.first_conv_node()
    c_out = getattr(model, name).conv_1.out_channels
    return (name,) + tuple(R.Conv1Pack(n, device, c_out) for n in n_nets)


def time_major_rows(seq_rows: torch.Tensor, t_idx: torch.Tensor, pitch: int | None = None) -> torch.Tensor:
    """Frame-table rows of the (t, b) frames in time-major order, for sequences of T frames whose rows start `pitch`
    rows apart (None: T, frame stacks stored as T consecutive rows; T + 3 for the windows of frame strips,
    R.sequence_rows): row = seq_rows[b] * pitch + t, with t_idx = arange(T).view(T, 1) (kept by the caller: no launch
    per step)."""
    pitch = t_idx.shape[0] if pitch is None else pitch
    return (seq_rows.view(1, -1) * pitch + t_idx).reshape(-1).contiguous()


# -- Learner.run: the Redis-facing edge ----------------------------------------------------------
def publishers(model, log_w, *pubs):
    """-> (`pubs` plus, when LOG_W is set, a checkpoint publisher of `model` — the tuple kept as
    `Learner._publishers` —, that checkpoint publisher or None).  Checkpoints go to ./weight/<ALG>/<time>/weight.pth
    (APE_X/Learner.py:256-262) once the snapshot's async D2H copy has landed."""
    path = wire.checkpoint_path(log_w)
    ckpt = ParamPublisher(model, None, None, None, on_ready=lambda sd, step: torch.save(sd, path)) if path else None
    return pubs + ((ckpt,) if ckpt else ()), ckpt


def check_served_fused(cfg, memory, fields=None) -> None:
    """What SERVED_FUSED_STEP needs, checked before the learner builds anything: FUSED_CONV1 (conv_1, or a RESCNN2D
    model's stem, reads the ring slot's frames through the frame table; the model itself is checked when the step
    state is built, require_fused_first_layer), a memory that binds ring slots (DeviceReplayClient.acquire / release), a
    ring whose minibatches hold BATCHSIZE records and, when `fields` is given, a ring that carries those fields."""
    if not cfg.FUSED_CONV1:
        raise ValueError("SERVED_FUSED_STEP reads the frames in the ring slot with the fused conv_1 or stem kernels: "
                         "it needs FUSED_CONV1")
    if not (hasattr(memory, "acquire") and hasattr(memory, "release")):
        raise TypeError("SERVED_FUSED_STEP needs a served memory that binds ring slots (DeviceReplayClient)")
    L = memory.ring.layout
    if L.batch != cfg.BATCHSIZE:
        raise ValueError(f"the server's ring holds minibatches of {L.batch}; the step graph is built for "
                         f"BATCHSIZE = {cfg.BATCHSIZE}")
    if fields is not None and [int(L.field_bytes[i]) for i in range(L.n_fields)] != [f.nbytes for f in fields]:
        raise ValueError("the server's ring does not carry this config's record fields (field sizes "
                         f"{[int(L.field_bytes[i]) for i in range(L.n_fields)]}, expected "
                         f"{[f.nbytes for f in fields]})")


class CapturedStep:
    """One learner step run eagerly or as a CUDA graph, on a stream of the learner's (Ape-X: the step's
    high-priority main stream; R2D2 / IMPALA: one stream of the step state).  Sets `_graph`, `_static` (the graph's
    output buffers), `_bound_warm` and `launches_per_step`; the learner initialises them to None, None, 0, None.

    The callers warm up before the capture in two ways, on purpose.  A step that draws its own minibatch (the
    in-process `fused_step`) runs its three warm-ups and the capture in its first call, under the replay's lock
    (bench.py's warm-up loop counts on "3 eager warm-ups + capture" in the first call).  A step on a served ring slot
    needs a new slot for each warm-up, so `_served_step` warms up over BOUND_WARMUP calls and captures on the next."""

    BOUND_WARMUP = 3       # eager steps on served minibatches before the bound step is captured

    def _served_step(self, body, use_graph: bool, stream):
        """One step on the slot `memory.acquire()` bound: the first BOUND_WARMUP calls run `body` eagerly on `stream`
        (lazy inits stay outside the capture), each on its own minibatch; the next call captures it; every later call
        replays the graph.  The caller releases the slot after this returns: the step is then enqueued."""
        if self._graph is not None:
            self._graph.replay()
            return self._static
        if use_graph and self._bound_warm < self.BOUND_WARMUP:
            self._bound_warm += 1
            return self._warm_up(body, 1, stream)
        return self._eager_or_captured(body, use_graph, stream)

    def _eager_or_captured(self, body, use_graph: bool, stream):
        """`body` (one step) run eagerly, its libb2rl launches counted into `launches_per_step`; or, with
        `use_graph`, captured on `stream` into `_graph`, whose launches are counted the same way, and replayed: every
        later step replays it.  -> the step's outputs (for the graph: `_static`, its static output buffers)."""
        lib = _lib.load()
        if not use_graph:
            c0 = lib.b2rl_launch_count()
            r = body()
            self.launches_per_step = lib.b2rl_launch_count() - c0
            return r
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        c0 = lib.b2rl_launch_count()
        with torch.cuda.graph(g, stream=stream):
            self._static = body()
        self.launches_per_step = lib.b2rl_launch_count() - c0   # recorded into the graph, replayed each step
        self._graph = g
        g.replay()
        return self._static

    def _warm_up(self, body, n: int, stream):
        """`n` eager runs of `body` on `stream`, so that lazy inits (cuDNN plans, optimizer state, workspaces)
        happen outside the capture.  -> what the last one returned."""
        cur = torch.cuda.current_stream(self.device)
        stream.wait_stream(cur)
        with torch.cuda.stream(stream):
            for _ in range(n):
                r = body()
        cur.wait_stream(stream)
        return r


class TargetNetLearner(CapturedStep):
    """The parts of `Learner` that Ape-X and R2D2 share (online + target network, run loop, write-back cadence,
    `Start` handshake, periodic log).  Uses the learner's `cfg`, `model`, `target_model`, `memory`, `_served`,
    `connect` and `writer`.  A learner provides `_next_step(step, log_every)` and sets `LOG_LINE`, its log line
    formatted with `last_log`, `num_memory` and `max_weight`; `PUBLISH_EVERY`, the steps between two publications
    of the online weights; and `LOG_STATS`, the names of the stats `_next_step` returns."""

    LOG_LINE: str
    PUBLISH_EVERY: int
    LOG_STATS: tuple

    def run(self, max_steps: int | None = None, log_every: int = 500):
        """Learner.run (APE_X/Learner.py:140-262, R2D2/Learner.py:217-339) with the reference's cadence: wait for
        more than BUFFER_SIZE records, announce `Start`, then per step `_next_step` (retried after 2 ms, and not
        counted, while no minibatch is ready: APE_X/Learner.py:166-170); hard target sync every TARGET_FREQUENCY
        steps (+ `target_state_dict`, APE_X/Learner.py:207-210); `state_dict` / `count` = step - 50 every
        PUBLISH_EVERY steps (:212-216; R2D2 publishes every 25 steps and still counts step - 50, sic
        R2D2/Learner.py:289-293); and every `log_every` (500) steps the `reward` drain + log line and a checkpoint
        of the online weights (APE_X/Learner.py:219-262, R2D2/Learner.py:296-339).  Publication and checkpoints go
        through ParamPublisher (async D2H into pinned memory), so none of them stalls the learner stream."""
        pub, pub_t, ckpt = self._start()
        step, acc, t0 = 0, None, time.time()
        self.last_log = None
        while max_steps is None or step < max_steps:
            tot = self._next_step(step + 1, log_every)
            if tot is None:
                time.sleep(0.002)
                continue
            step += 1
            acc = tot if acc is None else acc + tot
            if step % self.cfg.TARGET_FREQUENCY == 0:
                self.target_model.updateParameter(self.model, 1)
                pub_t.snapshot(step)                 # async D2H; published by a later poll()
            if step % self.PUBLISH_EVERY == 0:
                pub.snapshot(step - 50)
            for p in self._publishers:
                p.poll()
            if step % log_every == 0:
                self._log(step, log_every, t0, ckpt, **dict(zip(self.LOG_STATS, (acc / log_every).tolist())))
                acc, t0 = None, time.time()
        return step

    def _write_back(self, step: int, log_every: int, idx, prio) -> None:
        """The write-back cadence (APE_X/Learner.py:189-197, R2D2/Learner.py:266-274): every `log_every` steps the
        eviction request (`memory.lock`), which skips that step's write-back unless it has been served by then.  An
        in-process replay without a running ingest thread serves it inline; a served memory passes it on to its
        server.  `prio` None: the step has written its priorities back itself."""
        if step % log_every == 0:
            self.memory.lock = True
            if not self._served and (self.connect is None or not self.memory.is_alive()):
                self.memory._evict_on_request()
        if prio is not None and self.memory.lock is False:
            self.memory.update(idx, prio)

    @property
    def state_dict(self):
        return {k: v.cpu() for k, v in self.model.state_dict().items()}

    @property
    def target_state_dict(self):
        return {k: v.cpu() for k, v in self.target_model.state_dict().items()}

    def _start(self):
        """Learner.run's set-up (APE_X/Learner.py:140-155, R2D2/Learner.py:217-234): wait for more than BUFFER_SIZE
        records, publish the initial weights and announce `Start`, then build `_publishers`.
        -> (parameter publisher, target publisher, checkpoint publisher or None)"""
        while len(self.memory.memory) <= self.cfg.BUFFER_SIZE:
            time.sleep(0.05)
        if self.connect is not None:
            self.connect.set("state_dict", pickle.dumps(self.state_dict))
            self.connect.set("count", pickle.dumps(1))
            self.connect.set("target_state_dict", pickle.dumps(self.target_state_dict))
            self.connect.set("Start", pickle.dumps(True))
        pub = ParamPublisher(self.model, self.connect, "state_dict", "count")
        pub_t = ParamPublisher(self.target_model, self.connect, "target_state_dict", None)
        self._publishers, ckpt = publishers(self.model, self.cfg.LOG_W, pub, pub_t)
        return pub, pub_t, ckpt

    def _log(self, step, log_every, t0, ckpt, mean_value, norm, **stats) -> None:
        """The every-`log_every` tail (APE_X/Learner.py:219-262, R2D2/Learner.py:296-339): drain the actors'
        `reward` list, set `last_log` (+ `stats`), print LOG_LINE, write the TensorBoard scalars and snapshot a
        checkpoint (`ckpt`: the checkpoint publisher or None)."""
        reward, n_rew = wire.drain_rewards(self.connect) if self.connect is not None else (-21.0, 0)
        self.last_log = {"step": step, "mean_value": mean_value, "norm": norm, "reward": reward, **stats,
                         "time_per_step": (time.time() - t0) / log_every}
        mem = self.memory.memory
        print(self.LOG_LINE.format(num_memory=len(mem), max_weight=mem.max_weight, **self.last_log))
        if self.writer is not None:
            if n_rew:
                self.writer.add_scalar("Reward", reward, step)
            self.writer.add_scalar("value", mean_value, step)
            self.writer.add_scalar("norm", norm, step)
        if ckpt is not None:
            ckpt.snapshot(step)
