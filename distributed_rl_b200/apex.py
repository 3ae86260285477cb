"""Ape-X learner side: `Replay` and `Learner` with the reference's surface
(APE_X/ReplayMemory.py:19-167, APE_X/Learner.py:20-272) on top of the
HBM-resident replay and the fused kernels.

What changed relative to the reference, and why it is still a drop-in:
  * replay contents + priorities live in HBM (DeviceReplay); `Replay.sample()`
    returns the same 7-list `[s, a, r, s', done, w, idx]`, but as CUDA tensors,
    so `Learner.train` never copies frames host->device (the reference converts
    to fp32 on the CPU and ships 4x the bytes, APE_X/Learner.py:61-67).
  * `Learner.train` has no device->host sync: double-DQN argmax, target, clipped
    TD, priority, loss and dLoss/dQ come from one kernel (b2rl_apex_target) and
    the network backward is seeded with dLoss/dQ directly.
  * priorities are written back immediately (`Replay.update` enqueues the tree
    update on the stream) instead of after >1000 pending entries
    (APE_X/ReplayMemory.py:147-150); eviction is the ring's FIFO overwrite, so
    the `lock` flag handshake (:151-160, APE_X/Learner.py:189-197) is a no-op.
  * `Learner.fused_step()` runs sample -> gather -> 3 forwards -> target ->
    backward -> RMSprop -> priority write-back as one CUDA graph.
"""
from __future__ import annotations

import pickle
from dataclasses import dataclass, field

import numpy as np
import torch

from . import replay as R
from .agent import GraphAgent
from .learner_common import (Conv1Gathered as _Conv1Gathered, MemoryView, ReplayThread, TargetNetLearner,
                             _attach_replay, check_served_fused, conv1_packs, make_optimizer)


@dataclass
class ApexConfig:
    """The globals the reference lifts out of cfg/ape_x.json (configuration.py:39-98)."""
    BATCHSIZE: int = 32
    ACTION_SIZE: int = 6
    ALPHA: float = 0.6
    BETA: float = 0.4
    GAMMA: float = 0.99
    UNROLL_STEP: int = 3
    REPLAY_MEMORY_LEN: int = 100000
    BUFFER_SIZE: int = 50000
    TARGET_FREQUENCY: int = 2500
    LEARNER_DEVICE: str = "cuda:0"
    REDIS_SERVER: str = "localhost"
    LOG_W: str | None = None        # ./weight/<ALG>/<time> (configuration.py:101-109); None: no checkpoints
    OPTIM_INFO: dict = field(default_factory=lambda: {
        "name": "rmsprop", "lr": 0.0000625, "eps": 1.5e-7, "decay": 0, "alpha": 0.95, "momentum": 0,
        "centered": True})
    MODEL: dict = field(default_factory=lambda: default_apex_model())
    CHANNELS_LAST: bool = True      # NHWC activations/weights: cuDNN's TF32 kernels skip their layout transposes
    FUSED_CONV1: bool = True        # gather + conv_1 on the wgmma tensor cores (csrc/conv1.cu) in fused_step
    FUSED_OPTIM: bool = True        # RMSprop + zero_grad + grad-norm in one launch (csrc/optim.cu)
    EARLY_HEAD_UPDATE: bool = True  # RMSprop of the dense heads as soon as their gradients are final (no clipping in :123-138)
    CUDNN_BENCHMARK: bool = True    # let cuDNN time its conv_2/conv_3 algorithms once (no precision change)
    DEFERRED_WGRAD: bool = True      # weight gradients on a side stream, off the critical path of backward
    PARALLEL_FORWARDS: bool = True   # the three forward passes of a step on three streams (fork/join inside the graph)
    FUSED_DUELING_TAIL: bool = True  # heads' second layers + dueling combine in one kernel (csrc/dueling.cu)
    DENSE_3XTF32: bool = True       # dense heads as 3xTF32 wgmma GEMMs at fp32 accuracy (csrc/gemm.cu)
    BATCHED_ONLINE: bool = True     # the online net's two passes (s with grad, s' without) as ONE B = 2*BATCHSIZE call
    SERVED_FUSED_STEP: bool = False  # on a served replay (DeviceReplayClient), run() steps the captured fused step on
                                     # the bound ring slot instead of sample() -> train() -> update()
    FRAME_DEDUP: bool = False        # store every distinct frame once, in a pool of FRAMES_PER_TRANSITION frames per
                                     # slot (R.DedupReplay, DESIGN.md §4.16): samples are the same, the replay smaller
    FRAMES_PER_TRANSITION: float = 4.0
    DEDUP_WINDOW: int = 1 << 20      # a frame is reused only from the last DEDUP_WINDOW frames stored (at most 1/8 of
                                     # the pool, see dedup_geometry)
    FRAME_CODEC: bool = False        # store a FRAME_DEDUP store's frames losslessly encoded in a ring of bytes in HBM
                                     # (R.CodedDedupReplay, DESIGN.md §4.22).  Unlike R2D2's POOL_CODEC, which decodes
                                     # into a staged minibatch, the step still reads the pool in place: conv_1 decodes
                                     # the sampled frames on chip
    POOL_BYTES_PER_TRANSITION: float | None = None   # FRAME_CODEC's ring: this many bytes per slot (see pool_bytes);
                                                     # size it from CodedDedupReplay.codec_stats()

    def __post_init__(self):
        R.check_codec_keys(self, "FRAME_CODEC", "POOL_BYTES_PER_TRANSITION")

    @staticmethod
    def from_configuration():
        import configuration as C  # the drop-in module (dropin/configuration.py) or the user's own
        kw = {k: getattr(C, k) for k in ("BATCHSIZE", "ACTION_SIZE", "ALPHA", "BETA", "GAMMA", "UNROLL_STEP",
                                         "REPLAY_MEMORY_LEN", "BUFFER_SIZE", "TARGET_FREQUENCY",
                                         "LEARNER_DEVICE", "REDIS_SERVER", "OPTIM_INFO", "MODEL")}
        kw["LOG_W"] = getattr(C, "LOG_W", None)
        for k in ("FRAME_DEDUP", "FRAMES_PER_TRANSITION", "DEDUP_WINDOW", "FRAME_CODEC",
                  "POOL_BYTES_PER_TRANSITION"):                                # optional keys of cfg/ape_x.json
            if hasattr(C, k):
                kw[k] = getattr(C, k)
        return ApexConfig(**kw)


def dedup_geometry(cfg: ApexConfig) -> tuple:
    """(pool frames, window) of a FRAME_DEDUP replay: ceil(FRAMES_PER_TRANSITION * REPLAY_MEMORY_LEN) frames, and
    DEDUP_WINDOW capped at an eighth of them.  A slot stays live until pool - window frames have been stored after it,
    so the cap keeps that at least 7/8 of the pool: ~2.3 REPLAY_MEMORY_LEN records at the ~3 new frames per record
    the reference actor sends, more than the slot ring holds."""
    return R.dedup_pool_geometry(cfg.FRAMES_PER_TRANSITION, cfg.REPLAY_MEMORY_LEN, cfg.DEDUP_WINDOW)


def pool_bytes(cfg: ApexConfig) -> int | None:
    """Bytes of a FRAME_CODEC store's frame ring (None without FRAME_CODEC): R.coded_pool_bytes at
    POOL_BYTES_PER_TRANSITION bytes per slot, by default (F + 1) x 7 072 for dedup_geometry's F frames.  It must hold
    7 072 (W + 10) bytes whatever the frames (DESIGN.md §4.22)."""
    if not cfg.FRAME_CODEC:
        return None
    return R.coded_pool_bytes(cfg.FRAMES_PER_TRANSITION, cfg.REPLAY_MEMORY_LEN, cfg.POOL_BYTES_PER_TRANSITION)


def default_apex_model() -> dict:
    """The dueling DQN of cfg/ape_x.json:37-88 (values are configuration, not code)."""
    return {
        "module00": {"netCat": "CNN2D", "iSize": 4, "nLayer": 4, "fSize": [8, 4, 3, -1], "nUnit": [32, 64, 64],
                     "padding": [0, 0, 0], "stride": [4, 2, 1], "act": ["relu", "relu", "relu"],
                     "BN": [False] * 4, "linear": True, "input": [0], "prior": 0},
        "module02": {"netCat": "MLP", "iSize": 3136, "nLayer": 2, "fSize": [512, 6], "act": ["relu", "linear"],
                     "BN": [False] * 3, "prior": 1, "prevNodeNames": ["module00"]},
        "module02_1": {"netCat": "MLP", "iSize": 3136, "nLayer": 2, "fSize": [512, 1], "act": ["relu", "linear"],
                       "BN": [False] * 3, "prior": 1, "prevNodeNames": ["module00"]},
        "module03": {"netCat": "Add", "prior": 2, "prevNodeNames": ["module02", "module02_1"]},
        "module03_1": {"netCat": "Mean", "prior": 2, "prevNodeNames": ["module02"]},
        "module04": {"netCat": "Substract", "prior": 3, "prevNodeNames": ["module03", "module03_1"],
                     "output": True},
    }


class Replay(ReplayThread):
    """APE_X/ReplayMemory.py Replay (:19-167): same methods and attributes."""

    def __init__(self, cfg: ApexConfig | None = None, connect=None):
        super().__init__(cfg or ApexConfig.from_configuration(), connect)
        if self.cfg.FRAME_CODEC:
            self.store = R.CodedDedupReplay(self.cfg.REPLAY_MEMORY_LEN, *dedup_geometry(self.cfg), pool_bytes(self.cfg),
                                            device=self.device)
        elif self.cfg.FRAME_DEDUP:
            self.store = R.DedupReplay(self.cfg.REPLAY_MEMORY_LEN, *dedup_geometry(self.cfg), device=self.device)
        else:
            self.store = R.DeviceReplay(self.cfg.REPLAY_MEMORY_LEN, R.APEX_FIELDS, self.device)
        self.memory = MemoryView(self.store, self.cfg.BETA)

    # -- ingest: records are [s, a, R_n, s', done, prio] pickled by the actors ----
    def push_records(self, blobs) -> None:
        """PER.push (baseline/PER.py:69-75) for a list of pickled actor records
        (APE_X/Player.py:252-261): the raw blobs copied to the device once and decoded
        there (wire.WireIngest), or decoded on the host when the batch must take that
        path whole; then the store's push (leaf write / path refresh)."""
        if not blobs:
            return
        batch = self._wire_decode(blobs)
        if batch is not None:        # decoded on the device (wire.WireIngest)
            with self._lock:
                self.store.push([batch[k] for k in ("s", "ns", "a", "r", "d")], batch["p"])
            self.total_frame += len(blobs)
            return
        from .wire import decode_apex
        recs = [pickle.loads(b) for b in blobs]
        n = len(recs)
        st = self._staging(n)        # pinned, on the GPU's NUMA node: the H2D copy is a straight DMA
        decode_apex(recs, {k: st[k][:n].numpy() for k in ("s", "ns", "a", "r", "d", "p")})
        with self._lock:
            self.store.push([st[k][:n] for k in ("s", "ns", "a", "r", "d")], st["p"][:n])
            st["event"].record(torch.cuda.current_stream(self.device))
        self.total_frame += n

    def _wire_ingest(self):
        from .wire import WireIngest
        return WireIngest("apex", self.device)

    def _staging(self, n: int) -> dict:
        """One of two pinned staging sets (alternating), grown on demand; reused only after the copy that
        last read it has completed."""
        from .hostmem import pinned_empty
        if not hasattr(self, "_stages"):
            self._stages, self._stage_i = [None, None], 0
        self._stage_i ^= 1
        st = self._stages[self._stage_i]
        if st is not None:
            st["event"].synchronize()
        if st is None or st["cap"] < n:
            cap = max(n, 2 * (st["cap"] if st else 0), 64)
            shape = tuple(R.APEX_FIELDS[0].shape)
            st = {"cap": cap, "event": torch.cuda.Event(),
                  "s": pinned_empty((cap, *shape), torch.uint8, self.device),
                  "ns": pinned_empty((cap, *shape), torch.uint8, self.device),
                  "a": pinned_empty((cap,), torch.int32, self.device),
                  "r": pinned_empty((cap,), torch.float32, self.device),
                  "d": pinned_empty((cap,), torch.uint8, self.device),
                  "p": pinned_empty((cap,), torch.float32, self.device)}
            self._stages[self._stage_i] = st
        return st

    def push_arrays(self, s, ns, a, r, d, p) -> None:
        """Same ingest for already-decoded arrays (host pinned or device)."""
        with self._lock:
            self.store.push([s, ns, a, r, d], p)
        self.total_frame += int(torch.as_tensor(p).numel())

    def begin_ingest(self, s, ns, a, r, d) -> None:
        """Pipelined ingest, phase 1: retire the slots about to be overwritten and start the
        host->device copy on the ingest stream (overlaps the learner step in flight)."""
        with self._lock:
            self.store.push_begin([s, ns, a, r, d], int(torch.as_tensor(a).numel()))

    def commit_ingest(self, p) -> None:
        """Phase 2: wait for the copy, publish the new priorities (records become sampleable)."""
        with self._lock:
            self.store.push_commit(p)
        self.total_frame += int(torch.as_tensor(p).numel())

    def ingest(self, s, ns, a, r, d, p) -> None:
        """Steady-state ingest, one call per learner iteration (b2rl_replay_ingest_pipelined): the batch handed
        over by the previous call becomes sampleable, this one's host->device copy starts on the library's copy
        stream and overlaps the learner step that follows.  All arguments pinned host (or device) tensors."""
        with self._lock:
            self.store.ingest_pipelined([s, ns, a, r, d], p)
        self.total_frame += int(p.numel())

    # -- sampling -------------------------------------------------------------------
    def buffer(self, m: int = 1) -> None:
        """Replay.buffer (:61-116): sample m*BATCHSIZE, IS weights, assemble minibatches."""
        B = self.cfg.BATCHSIZE
        with self._lock:
            idx, _, w = self.store.sample(B * m, beta=self.cfg.BETA)
            batch = self.store.gather(idx)
        for k in range(m):
            sl = slice(k * B, (k + 1) * B)
            self.deque.append([batch["state"][sl], batch["action"][sl], batch["reward"][sl],
                               batch["next_state"][sl], batch["done"][sl], w[sl], idx[sl]])

    def _update(self):
        """Replay._update (:49-59) applies the pending write-backs; here update() has already enqueued them on
        the stream, so all that is left is to make them visible to the host."""
        torch.cuda.current_stream(self.device).synchronize()


class _StepState:
    """What `Learner.fused_step` keeps from one step to the next: its streams and fork/join sites, the conv_1 weight
    packs, the weight-gradient sink, the draw buffers and the batched pass's conv_1 output.  Built once, before the
    first step's warm-up, so that no stream, event or buffer is created inside the warm-up or the capture.

    Stream priorities are captured into the graph's kernel nodes: the main branch runs at -2 and so does the target
    network's pass (both feed the target kernel); the operand packs and the side branch (needed much later) at 0;
    the sink's lanes at -1 (convolutions) and 0 (heads)."""

    def __init__(self, L: "Learner"):
        from .linear import SideBranch, WeightGradSink
        cfg, dev, B = L.cfg, L.device, L.cfg.BATCHSIZE
        self.main = torch.cuda.Stream(dev, priority=-2)
        packs, target = torch.cuda.Stream(dev), torch.cuda.Stream(dev, priority=-2)

        def branch(stream):          # without PARALLEL_FORWARDS the step runs on one stream
            return SideBranch(stream if cfg.PARALLEL_FORWARDS else None)
        self.conv1_packs = branch(target)         # conv_1 waits for this launch
        self.head_packs_built = branch(packs)
        self.target_pass = branch(target)
        self.side = branch(packs)                 # Q_online(s') or the batched pass's action / done conversion; W^T pack
        self.prio_update = branch(target)
        self.max_w = SideBranch(packs)            # data parallel: the reduced max IS weight, for the next step
        self.head_packs = None                    # (online, target) heads' forward operands of this step
        self.resident = None                      # (online, target) heads' persistent operand images, or None
        self.pack1 = self.pack2 = self.cur = self.y_big = self.sink = self.frames = None
        if not L._conv1_ready():
            if L._served:
                raise ValueError("SERVED_FUSED_STEP reads the ring slot's frames with the fused conv_1 kernels: the "
                                 "model's first node must be the Atari conv_1")
            return
        # pack1: online net (grad pass on s); pack2: online + target in one pass over s'
        self.conv_name, self.pack1, self.pack2 = conv1_packs(L.model, dev, 1, 2)
        idx_w = dict(idx=torch.empty(B, dtype=torch.int64, device=dev), w=torch.empty(B, dtype=torch.float32, device=dev))
        if L._served:
            # The draw is the server's.  Before each step, memory.acquire() binds a filled ring slot to these buffers
            # (outside the graph): its header, idx, w, action, reward and done are copied in, and the two entries of
            # `table` receive the addresses of its state / next_state rows, which conv_1 reads in place.
            self.cur = dict(R.alloc_rows(R.APEX_FIELDS, B, dev, ("action", "reward", "done")), **idx_w,
                            header=torch.zeros(2, dtype=torch.int64, device=dev))
            self.table = torch.zeros(2, dtype=torch.int64, device=dev)
            self.frames = {"state": R.BoundFrames(self.table, 0, B), "next_state": R.BoundFrames(self.table, 1, B)}
        else:
            self.cur = dict(L.memory.store.alloc_batch(B, ("action", "reward", "done")), **idx_w)
        if cfg.PARALLEL_FORWARDS and cfg.BATCHED_ONLINE:
            self.y_big = torch.empty((3, B, 20, 20, self.pack1.c_out), dtype=torch.float32, device=dev)
        if L._fused_optim:
            # The heads' operand images live across steps: the fused optimizer rewrites the online ones whenever it
            # steps the weights, and the target's change only at a target sync (GraphAgent.updateParameter repacks
            # them).  torch.optim cannot maintain them: that configuration packs them every step.
            on = L.model.keep_resident_heads(transposed=True)
            tg = L.target_model.keep_resident_heads(transposed=False)
            for group, ws in L.model.head_pieces():
                off = 0
                for w in ws:
                    L.optim.write_images(w, on[group]["fwd"], on[group]["bwdT"],
                                         sum(v.shape[0] for v in ws), off)
                    off += w.shape[0]
            self.resident = (on, tg) if on else None
        if cfg.DEFERRED_WGRAD and L._fused_optim:
            self.sink = WeightGradSink(dev)
            self.sink.grads_are_zero = True      # grads are pre-allocated and zeroed by the fused optimizer
            getattr(L.model, self.conv_name).split_backward = True
            if L._world > 1:
                L._bucket.attach_sink(self.sink)
            # Learner.step (:123-138) has no clipping: a parameter can be stepped once its own gradient is final
            # (after its all-reduce when data parallel).  The heads (97 % of the elements) are final ~150 us
            # before the conv stack's.
            self.early_params = [p for n, p in L.model.named_parameters() if not n.startswith(self.conv_name + ".")]
            self.early_ok = (cfg.EARLY_HEAD_UPDATE and bool(self.early_params)
                             and L.optim.set_early(self.early_params))


class Learner(TargetNetLearner):
    """APE_X/Learner.py Learner (:20-272): train / step / run / state_dict."""

    LOG_LINE = ("step:{step} // mean_value:{mean_value:.3f} // norm: {norm:.3f} // REWARD:{reward:.3f} // "
                "NUM_MEMORY:{num_memory} // Mean_Weight:{mean_weight:.3f} // MAX_WEIGHT:{max_weight:.3f} // "
                "TIME:{time_per_step:.5f} // loss:{loss:.5f}")
    PUBLISH_EVERY = 50
    LOG_STATS = ("loss", "mean_value", "mean_weight", "norm")

    def __init__(self, cfg: ApexConfig | None = None, connect=None, start_replay: bool = True,
                 writer=None, memory=None):
        """`memory`: a replay served from another process (replay_server.DeviceReplayClient, or anything with the
        `Replay` surface: sample / update / lock / memory).  run() then drives sample() -> train() -> update() with
        the reference's cadence (APE_X/Learner.py:163-197); without it the learner owns its replay and run() steps
        with fused_step().  With SERVED_FUSED_STEP, run() over a served memory steps fused_step() instead, on the
        slot `memory.acquire()` binds (same cadence): see _next_step."""
        self.cfg = cfg or ApexConfig.from_configuration()
        if memory is not None and self.cfg.SERVED_FUSED_STEP:
            check_served_fused(self.cfg, memory)
        self.device = torch.device(self.cfg.LEARNER_DEVICE)
        if self.cfg.CUDNN_BENCHMARK and self.device.type == "cuda":
            torch.backends.cudnn.benchmark = True
        self.build_model()
        self.build_optim()
        self.connect = connect
        self.memory = _attach_replay(self, memory, lambda: Replay(self.cfg, connect), connect, start_replay, wipe=True)
        self.writer = writer
        self.gamma_n = float(np.float32(0.99 ** self.cfg.UNROLL_STEP))  # hard-coded 0.99, :103
        self._graph = None
        self._fused = None              # _StepState, built by the first fused_step / _forward_backward_fused
        self._bound_warm = 0            # eager warm-up steps _bound_step has run
        self._world = 1
        self.launches_per_step = None   # libb2rl kernels per fused step (bench.py's gpu_launches)

    def enable_data_parallel(self):
        """Replay-sharded data parallelism (SURVEY.md §8e): every rank owns a replay shard and
        samples locally; per step one NCCL all-reduce (AVG) of the gradients, kept in ONE flat
        bucket so it is a single collective, and one MAX all-reduce of the max IS weight."""
        if self._served and self.cfg.SERVED_FUSED_STEP:
            raise ValueError("data parallelism samples every rank's own replay shard; a learner stepping served "
                             "minibatches (SERVED_FUSED_STEP) has no shard")
        from . import dist as D
        self._D = D
        self._world = D.world()
        self._bucket = D.FlatGradBucket(self.model.getParameters(), self.device,
                                        symmetric=D.PeerAllReduce.available(self.device))
        # the dense heads hold 97 % of the parameters and their gradients are complete first in the
        # backward pass: their all-reduce overlaps the backward of the convolution stack
        import os
        heads = [p for p in self.model.getParameters() if p.dim() == 2]
        if os.environ.get("B2RL_NO_OVERLAP"):
            heads = []
        self._bucket.enable_overlap(heads)
        # What is left after backward (the convolution stack's 0.3 MB) is the collective on the critical path: one
        # libb2rl kernel over NVLink peer memory instead of an NCCL launch (csrc/peer.cu; NCCL stays where peer
        # mapping is not available).  (A second overlapped NCCL group for conv_2 / conv_3 was tried: its kernel
        # cannot get SMs while the SM-filling conv_1 weight-gradient kernel runs, so it only added a launch.)
        self.peer_allreduce = self._bucket.enable_peer_allreduce()
        self.peer_allreduce_heads = getattr(self._bucket, "_peer_big", None) is not None
        self._max_w = torch.empty(1, dtype=torch.float32, device=self.device)       # being reduced this step
        self._max_w_use = None                                                      # reduced last step, used now

    def build_model(self):
        self.model = GraphAgent(self.cfg.MODEL).to(self.device)
        self.target_model = GraphAgent(self.cfg.MODEL).to(self.device)
        self._mf = torch.channels_last if self.cfg.CHANNELS_LAST else torch.contiguous_format
        if self.cfg.CHANNELS_LAST:
            self.model.to(memory_format=torch.channels_last)
            self.target_model.to(memory_format=torch.channels_last)
            if self.cfg.FUSED_CONV1:
                # conv_1 runs in libb2rl's kernels, which take the plain (c_out, 4, 8, 8) layout: keeping that weight
                # channels_last cost one re-layout copy per pack (three launches per step)
                for m in (self.model, self.target_model):
                    name = m.first_conv_node()
                    if name is not None and getattr(m, name).is_atari_conv1():
                        w = getattr(m, name).conv_1.weight
                        w.data = w.data.contiguous(memory_format=torch.contiguous_format)
        self.model.dense_3xtf32 = self.target_model.dense_3xtf32 = bool(self.cfg.DENSE_3XTF32)
        self.model.fused_dueling_tail = self.target_model.fused_dueling_tail = bool(self.cfg.FUSED_DUELING_TAIL)

    def build_optim(self):
        info = self.cfg.OPTIM_INFO
        fusable = (self.cfg.FUSED_OPTIM and info["name"] == "rmsprop" and not info.get("momentum", 0)
                   and not info.get("decay", 0) and self.device.type == "cuda")
        if fusable:
            from .optim import FusedRMSprop, flat_grads
            self._grad_flat = flat_grads(self.model.getParameters())     # adjacent head gradients: see linear._stacked_rows
            self.optim = FusedRMSprop(self.model.getParameters(), lr=info["lr"], alpha=info.get("alpha", 0.99),
                                      eps=info.get("eps", 1e-5), centered=info.get("centered", False))
        else:
            self.optim = make_optimizer(info, self.model.getParameters())
        self._fused_optim = fusable

    # -- one training step on an explicit minibatch (reference signature) -----------
    def _to_dev(self, x, dtype):
        if torch.is_tensor(x):
            return x.to(device=self.device, dtype=dtype, non_blocking=True)
        if isinstance(x, np.ndarray) and x.dtype == object:
            x = x.astype(np.float64 if dtype.is_floating_point else np.int64)
        return torch.as_tensor(x).to(device=self.device, dtype=dtype, non_blocking=True)

    def _forward_backward(self, state, action, reward, next_state, done, weight):
        s = (state.to(torch.float32) / 255.0).contiguous(memory_format=self._mf)        # :61-63, on the device
        ns = (next_state.to(torch.float32) / 255.0).contiguous(memory_format=self._mf)  # :65-67
        q = self.model.forward([s])[0]                 # :78
        with torch.no_grad():
            qn_target = self.target_model.forward([ns])[0]   # :85
            qn_online = self.model.forward([ns])[0]          # :87
        notdone = 1.0 - done.to(torch.float32)         # :76
        out = R.apex_target(q.detach(), qn_online, qn_target, action, reward, notdone, weight,
                            self.gamma_n, self.cfg.ALPHA)
        q.backward(out["grad_q"])                      # == loss.backward(), :112-115
        if self._world > 1:
            self._bucket.finish()
        return out

    def train(self, transition, t=0):
        state, action, reward, next_state, done, weight, idx = transition
        state = self._to_dev(state, torch.uint8)
        next_state = self._to_dev(next_state, torch.uint8)
        action = self._to_dev(action, torch.int64)
        reward = self._to_dev(reward, torch.float32)
        done = self._to_dev(done, torch.uint8) if not (torch.is_tensor(done) and done.dtype == torch.bool) \
            else done.to(self.device, torch.uint8)
        weight = self._to_dev(weight, torch.float32)
        out = self._forward_backward(state, action, reward, next_state, done, weight)
        info = self.step()
        info["mean_value"] = out["scalars"][1]
        info["loss"] = out["scalars"][0]
        return info, out["prio"], idx, out["scalars"][2]

    def step(self):
        """Learner.step (:123-138): 'norm' = sqrt(sum_i ||g_i||_2) (sic), RMSprop, zero_grad."""
        if self._fused_optim:
            return {"p_norm": self.optim.step(want_norm=True)[0]}    # update + zero_grad + norm: one launch
        grads = [p.grad for p in self.model.parameters() if p.grad is not None]
        p_norm = torch.stack(torch._foreach_norm(grads, 2)).sum().sqrt()
        self.optim.step()
        self.optim.zero_grad(set_to_none=False)
        return {"p_norm": p_norm}

    # -- fused gather + conv_1 path ------------------------------------------------------------
    def _conv1_ready(self) -> bool:
        return bool(self.cfg.FUSED_CONV1) and self.model.first_conv_node() is not None

    def _fused_state(self) -> "_StepState":
        if self._fused is None:
            self._fused = _StepState(self)
        return self._fused

    _pack2 = property(lambda self: self._fused_state().pack2)   # conv_1 weights of online + target, packed
    _cur = property(lambda self: self._fused.cur)      # the draw of the last fused_step: idx, w, action, reward, done

    def _pack_weights(self):
        """This step's weight packs.  They depend only on the weights, so they are forked at the start of the step
        and overlap the tree sample + scalar gather: the conv_1 packs (one launch; conv_1 waits for it, so it runs on
        the high-priority stream) and, for the batched online pass, the heads' forward operands of both networks
        (four 3136 x 512 matrices -> two packed images, needed ~120 us into the step)."""
        s = self._fused
        w_on = getattr(self.model, s.conv_name).conv_1.weight
        w_tg = getattr(self.target_model, s.conv_name).conv_1.weight
        with s.conv1_packs.fork():
            R.conv1_pack_jobs([(s.pack1, 0, w_on), (s.pack2, 0, w_on), (s.pack2, 1, w_tg)])   # one launch
        if s.resident is not None:
            s.head_packs = s.resident
        elif self.cfg.PARALLEL_FORWARDS and self.cfg.BATCHED_ONLINE:
            with s.head_packs_built.fork():
                with self.model.packed_heads_cache():
                    on = self.model.prepack_heads()
                with self.target_model.packed_heads_cache():      # was ~11 us in front of the target pass's GEMM
                    tg = self.target_model.prepack_heads()
            s.head_packs = (on, tg)

    def _forward_backward_fused(self, idx, action, reward, done, weight, prepacked=False, update_tree=False,
                                early_update=False):
        """Same maths as _forward_backward, but s and s' are never staged as uint8/fp32 batches:
        conv_1 reads the sampled rows straight from the replay payload (b2rl_conv1_fused).
        `prepacked`: the caller has already issued this step's _pack_weights().
        `update_tree`: write the new priorities back on a side stream as soon as the target kernel has produced
        them (overlapping backward); the caller then joins `prio_update` instead of calling store.update.
        `early_update`: the caller WILL call self.step() next; the heads' part of that optimizer step may then be
        issued here, behind their weight gradients on the sink's lane, while the conv stack's backward still runs."""
        s = self._fused_state()
        if self._served:        # the bound ring slot: its rows are the draws, in order
            st, src_s, src_ns, rows = None, s.frames["state"], s.frames["next_state"], None
        else:
            st = self.memory.store
            src_s, src_ns, rows = st.frame_source("state"), st.frame_source("next_state"), idx
        w_on = getattr(self.model, s.conv_name).conv_1.weight
        if not prepacked:
            self._pack_weights()
        s.conv1_packs.join()
        notdone = None
        batched = self.cfg.PARALLEL_FORWARDS and self.cfg.BATCHED_ONLINE
        resident = s.resident is not None
        on_packs, tg_packs = s.head_packs if (batched or resident) else (None, None)
        with self.model.packed_heads_cache(on_packs):   # online weights packed once
            if batched:
                # Q(s) (with grad) and Q_online(s') (without) share the online weights: every kernel after conv_1 is
                # launch / set-up bound at B = 512 (DESIGN.md §6b), so both run as ONE B = 2*BATCHSIZE pass
                # (conv_2, conv_3, heads' GEMM, dueling tail: one launch each instead of two).  The pass is recorded
                # on an OutputTape; the autograd graph of the s half is then built by replaying the recorded per-op
                # outputs (first B rows: views, no kernels) through the same forward code.  Q_target(s') runs
                # beside it on a second stream.
                from .linear import OutputTape
                B, c_out = weight.numel(), s.pack1.c_out
                big = s.y_big          # [0] conv_1(s) online, [1] conv_1(s') online, [2] conv_1(s') target
                if big.shape[1] != B:
                    raise ValueError(f"the batched online pass is sized for BATCHSIZE = {big.shape[1]}, got {B} rows")
                with torch.no_grad():
                    R.conv1_fused(src_s, rows, s.pack1, relu=True, out=big[0:1])
                    y_tg = R.conv1_fused(src_ns, rows, s.pack2, relu=True, out=big[1:3])[1]
                s.head_packs_built.join()      # long done; the heads' GEMM is ~100 us away
                with torch.no_grad():
                    with s.target_pass.fork(), self.target_model.packed_heads_cache(tg_packs):
                        qn_target = self.target_model.forward_from_conv1(y_tg, True)[0]  # :85
                    with s.side.fork():
                        if action.dtype != torch.int64:            # int32 replay field -> the target kernel's int64:
                            action = action.to(torch.int64)        # off the main branch (it sat in front of conv_1)
                        notdone = 1.0 - done.to(torch.float32)     # likewise (two launches in front of the target kernel)
                        if not resident:
                            self.model.prepack_heads(transposed=True)   # W^T operand of the heads' dgrad, off the main branch
                    y_both = big[0:2].view(2 * B, 20, 20, c_out).permute(0, 3, 1, 2)     # logical NCHW, physical NHWC
                    with OutputTape.record() as tape:
                        q_all = self.model.forward_from_conv1(y_both, True)[0]          # :78 and :87 in one pass
                qn_online = q_all[B:]
                y = _Conv1Gathered.apply(w_on, src_s, rows, s.pack1, self._mf, st, big[0].permute(0, 3, 1, 2), True)
                with OutputTape.replay(tape.half(B)):
                    q = self.model.forward_from_conv1(y, True)[0]                       # graph only: outputs replayed
            else:
                # Three separate passes, independent until the target kernel.  With PARALLEL_FORWARDS the two over s'
                # fork onto two streams (parallel branches of the step's CUDA graph) so their small kernels overlap.
                if not resident:
                    self.model.prepack_heads()
                with torch.no_grad():
                    y_on, y_tg = R.conv1_fused(src_ns, rows, s.pack2, relu=True)
                    with s.side.fork():
                        qn_online = self.model.forward_from_conv1(y_on, True)[0]        # :87
                        if self.cfg.PARALLEL_FORWARDS and not resident:   # on one stream backward packs it beside its wgrad lanes
                            self.model.prepack_heads(transposed=True)   # W^T operand of the heads' dgrad, off the main branch
                    with s.target_pass.fork(), self.target_model.packed_heads_cache(tg_packs):
                        qn_target = self.target_model.forward_from_conv1(y_tg, True)[0]  # :85
                y = _Conv1Gathered.apply(w_on, src_s, rows, s.pack1, self._mf, st, None, True)
                q = self.model.forward_from_conv1(y, True)[0]                        # :78 (ReLU in the conv_1 epilogue)
            s.side.join()
            s.target_pass.join()
        if notdone is None:
            notdone = 1.0 - done.to(torch.float32)
        out = R.apex_target(q.detach(), qn_online, qn_target, action, reward, notdone, weight,
                            self.gamma_n, self.cfg.ALPHA)
        if update_tree:      # priority write-back (one CTA) next to backward instead of after the optimizer
            with s.prio_update.fork():
                st.update(idx, out["prio"])
        sink = s.sink
        if sink is None:
            q.backward(out["grad_q"])
        else:
            with sink.active():
                q.backward(out["grad_q"])
            if early_update and s.early_ok and all(id(p) in sink.accumulated[0] for p in s.early_params):
                if self._world > 1:
                    # data parallel: the heads' all-reduce was launched from this lane when their last gradient
                    # landed; the lane waits for it, then steps them — still beside the conv stack's backward
                    sink.run_on_lane(lambda: self._bucket.wait_group(0) and self.optim.step_early(), 0)
                else:
                    sink.run_on_lane(self.optim.step_early, 0)
            sink.join()
        if self._world > 1:
            self._bucket.finish()
        return out

    # -- the whole hot loop iteration as one CUDA graph -----------------------------------
    def fused_step(self, use_graph: bool = True):
        """sample -> gather -> forwards -> target -> backward -> RMSprop -> priority
        write-back (APE_X/Learner.py:165-197) with no host round trip.  On a served memory (SERVED_FUSED_STEP) the
        same step on the slot the last `memory.acquire()` bound; see _bound_step."""
        if self._graph is not None:
            self._graph.replay()
            return self._static
        if self._served:
            if not self.cfg.SERVED_FUSED_STEP:
                raise RuntimeError("fused_step() samples the learner's own replay; a served replay is driven by run() "
                                   "(or set SERVED_FUSED_STEP)")
            return self._bound_step(use_graph)
        B = self.cfg.BATCHSIZE
        st = self.memory.store
        s = self._fused_state()
        fused_conv1 = s.pack1 is not None
        side = fused_conv1 and self.cfg.PARALLEL_FORWARDS
        batched = side and self.cfg.BATCHED_ONLINE      # the batched pass converts the action itself

        def body():
            max_w, mw_work = None, None
            if self._world > 1:
                # priority-max reduction: IS weights are normalised by the GLOBAL max weight.  The MAX
                # all-reduce of this step's local value runs behind the step and is used by the next one
                # (the reference's own max_weight is up to 16 minibatches stale, APE_X/ReplayMemory.py:61-67).
                mw_work = self._D.all_reduce_max_(st.max_weight(self.cfg.BETA, out=self._max_w), async_op=True)
                max_w = self._max_w_use
            if fused_conv1:
                self._pack_weights()
                # ONE launch draws the minibatch: indices + IS weights from the sum-tree and the sampled slots'
                # scalar fields (a, r, done); the frames are read in place by the conv_1 kernels.
                # (Drawing the NEXT minibatch at the end of the step would hide these ~5 us too, but a ring slot
                # overwritten by the ingest between the draw and its use would pair new frames with the old
                # record's a / r / done — DESIGN.md §4.2.)
                c = s.cur
                st.sample_fetch(B, self.cfg.BETA, c["idx"], c["w"], {k: c[k] for k in ("action", "reward", "done")},
                                max_w=max_w)
                idx = c["idx"]
                out = self._forward_backward_fused(idx, c["action"] if batched else c["action"].to(torch.int64),
                                                   c["reward"], c["done"], c["w"],
                                                   prepacked=True, update_tree=side, early_update=True)
            else:
                idx, _, w = st.sample(B, beta=self.cfg.BETA, want_prob=False, max_w=max_w)
                b = st.gather(idx)
                out = self._forward_backward(b["state"], b["action"].to(torch.int64), b["reward"],
                                             b["next_state"], b["done"], w)
            info = self.step()
            if side:
                s.prio_update.join()
            else:
                st.update(idx, out["prio"])
            if mw_work is not None:
                # the reduced maximum becomes the NEXT step's normaliser: wait + copy on a side stream (this step's
                # draw has long read the old value), joined here at no cost instead of 5 us at the end of the step
                with s.max_w.fork(after_current=False):
                    mw_work.wait()
                    self._max_w_use.copy_(self._max_w)
                s.max_w.join()
            return {"scalars": out["scalars"], "p_norm": info["p_norm"], "prio": out["prio"], "idx": idx}

        if self._world > 1 and self._max_w_use is None:      # first step: reduce synchronously once
            self._max_w_use = self._D.all_reduce_max_(st.max_weight(self.cfg.BETA)).clone()
        # The step is warmed up and captured on its HIGH-priority main stream (kernel nodes inherit it): the side
        # branches (weight gradients, early optimizer step, operand packs) only fill SMs the critical chain leaves idle.
        if not use_graph:
            return self._eager_or_captured(body, False, s.main)
        self.optim.zero_grad(set_to_none=False)
        # The ingest thread keeps pushing on the same replay handle: hold its lock so that no cudaMalloc /
        # cudaHostAlloc / copy of that thread lands inside the warm-up or the (global-mode) capture.
        with self.memory._lock:
            self._warm_up(body, 3, s.main)
            return self._eager_or_captured(body, True, s.main)

    def _bound_step(self, use_graph: bool = True):
        """One step on the served minibatch `memory.acquire(cur, frames)` bound: fused_step's graph, with the draw
        (sample_fetch) and the in-graph tree update replaced by reads of the bound buffers; the priorities leave
        through memory.update() after the step.  Warm-up, capture and replay: CapturedStep._served_step, on the main
        stream."""
        s = self._fused_state()
        c = s.cur
        batched = self.cfg.PARALLEL_FORWARDS and self.cfg.BATCHED_ONLINE   # the batched pass converts the action

        def body():
            self._pack_weights()
            out = self._forward_backward_fused(c["idx"], c["action"] if batched else c["action"].to(torch.int64),
                                               c["reward"], c["done"], c["w"], prepacked=True, early_update=True)
            info = self.step()
            return {"scalars": out["scalars"], "p_norm": info["p_norm"], "prio": out["prio"], "idx": c["idx"]}

        if use_graph and self._bound_warm == 0:
            self.optim.zero_grad(set_to_none=False)
        return self._served_step(body, use_graph, s.main)

    # -- one step of run() ---------------------------------------------------------------------------
    def _next_step(self, step: int, log_every: int):
        """One iteration of the reference loop (APE_X/Learner.py:163-197) and its write-back cadence.  In-process:
        fused_step(), whose graph writes the priorities back.  Served: a minibatch from `memory`, then the
        write-back; with SERVED_FUSED_STEP the oldest filled slot is bound (memory.acquire), fused_step() runs on it
        and the slot is handed back once the step is enqueued (memory.release: conv_1's weight gradient, in
        backward, is its last reader); otherwise sample() -> train().
        -> {loss, mean(y), mean(w), norm} as a device tensor, or None when no minibatch is ready."""
        if self._served and not self.cfg.SERVED_FUSED_STEP:
            batch = self.memory.sample()
            if batch is False:
                return None
            info, prio, idx, mean_w = self.train(batch)
            tot = torch.stack([info["loss"], info["mean_value"], mean_w, info["p_norm"].reshape(())])
        else:
            if self._served:
                s = self._fused_state()
                if self.memory.acquire(s.cur, s.frames) is None:
                    return None
                out = self.fused_step()
                self.memory.release()
                idx, prio = out["idx"], out["prio"]
            else:
                out = self.fused_step()
                idx, prio = None, None
            tot = torch.cat([out["scalars"], out["p_norm"].reshape(1)])
        self._write_back(step, log_every, idx, prio)
        return tot

