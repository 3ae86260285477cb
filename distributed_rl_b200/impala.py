"""IMPALA learner side with the reference's surface (IMPALA/ReplayMemory.py:14-85,
IMPALA/Learner.py:17-297).  Rollouts (T+1 frames, T actions / behaviour probs /
rewards, done) live in HBM; sampling is uniform WITHOUT replacement per call like
baseline/utils.py ReplayMemory.sample (:310-315); the V-trace backward scan
(:176-200, a Python loop of ~10 tiny kernels per step in the reference) is one
launch of b2rl_vtrace."""
from __future__ import annotations

from dataclasses import dataclass, field

import torch

from . import replay as R
from .agent import GraphAgent
from .learner_common import (CapturedStep, Conv1Gathered, ReplayThread, StemGathered, _attach_replay,
                             check_served_fused, conv1_packs, fused_first_layer, make_optimizer, publishers,
                             time_major_rows)
from .publish import ParamPublisher


def default_impala_model() -> dict:
    """cfg/impala.json:24-52 (configuration values)."""
    return {
        "module00": {"netCat": "CNN2D", "iSize": 4, "nLayer": 3, "fSize": [8, 4, -1], "nUnit": [16, 32],
                     "padding": [0, 0], "stride": [4, 2], "act": ["relu", "relu"], "BN": [False] * 3,
                     "linear": True, "input": [0], "prior": 0},
        "module01": {"netCat": "MLP", "iSize": 2592, "nLayer": 2, "fSize": [256, 7], "act": ["relu", "linear"],
                     "BN": [False, False], "prior": 1, "prevNodeNames": ["module00"], "output": True},
    }


def resnet_small_model() -> dict:
    """The IMPALA paper's residual network (Espeholt et al. 2018, Fig. 3, without the LSTM) in the same graph form:
    a RESCNN2D node (three sections of conv, max-pool and two residual blocks at 16, 32, 32 channels; 84 -> 42 -> 21
    -> 11) and the MLP head 3 872 -> 256 (ReLU) -> 7.  1 090 368 parameters.  ImpalaConfig(MODEL=resnet_small_model())
    trains it; with FUSED_CONV1 its stem (first conv + max-pool) reads the frames in place (csrc/stem.cu)."""
    return {
        "module00": {"netCat": "RESCNN2D", "iSize": 4, "nUnit": [16, 32, 32], "blockNum": 2, "linear": True,
                     "input": [0], "prior": 0},
        "module01": {"netCat": "MLP", "iSize": 3872, "nLayer": 2, "fSize": [256, 7], "act": ["relu", "linear"],
                     "BN": [False, False], "prior": 1, "prevNodeNames": ["module00"], "output": True},
    }


@dataclass
class ImpalaConfig:
    BATCHSIZE: int = 32
    ACTION_SIZE: int = 6
    GAMMA: float = 0.99
    C_LAMBDA: float = 1
    C_VALUE: float = 1.0
    P_VALUE: float = 1.0
    ENTROPY_R: float = 0.01
    UNROLL_STEP: int = 20
    REPLAY_MEMORY_LEN: int = 10000
    BUFFER_SIZE: int = 9999
    LEARNER_DEVICE: str = "cuda:0"
    REDIS_SERVER: str = "localhost"
    LOG_W: str | None = None
    OPTIM_INFO: dict = field(default_factory=lambda: {"name": "rmsprop", "lr": 6e-4, "decay": 0})
    MODEL: dict = field(default_factory=default_impala_model)
    FUSED_CONV1: bool = True     # conv_1 (4 -> 16 channels) of every frame through libb2rl's wgmma kernel; with a
                                 # RESCNN2D model (resnet_small_model), its stem through libb2rl's stem kernels
    DENSE_3XTF32: bool = True    # the head's first layer (2592 -> 256; 3872 -> 256 for resnet_small_model) as a 3xTF32
                                 # wgmma GEMM (csrc/gemm.cu) instead of an fp32 SIMT sgemm
    SERVED_FUSED_STEP: bool = False  # on a served replay (DeviceReplayClient), run() steps a captured step on the
                                     # bound ring slot instead of sample() -> train()
    FRAME_DEDUP: bool = False    # store every distinct frame once, in a pool of FRAMES_PER_ROLLOUT frames per slot
                                 # (R.RolloutDedupReplay, DESIGN §4.20): overlapping stacks, the bootstrap stack and
                                 # the padding of short rollouts share their frames.  Draws and samples are a stack
                                 # store's.
    FRAMES_PER_ROLLOUT: float = 24.0
    DEDUP_WINDOW: int = 1 << 14  # a frame is reused only from the last DEDUP_WINDOW frames stored (at most 1/8 of the
                                 # pool, see dedup_geometry)
    STAGED_POOL_CODEC: bool = False  # store a FRAME_DEDUP store's frames losslessly encoded in a ring of bytes in HBM
                                     # (DESIGN §4.23); each step decodes the drawn rollouts' distinct frames into a
                                     # staged frame pool that conv_1 reads, as R2D2's POOL_CODEC decodes into a staged
                                     # batch.  Not named POOL_CODEC: IMPALA's staged pool is a plane table, not a batch.
    POOL_BYTES_PER_ROLLOUT: float | None = None    # STAGED_POOL_CODEC's ring: this many bytes per slot (pool_bytes);
                                                   # size it from RolloutDedupReplay.codec_stats()

    def __post_init__(self):
        R.check_codec_keys(self, "STAGED_POOL_CODEC", "POOL_BYTES_PER_ROLLOUT")

    @staticmethod
    def from_configuration():
        import configuration as C
        names = ("BATCHSIZE", "ACTION_SIZE", "GAMMA", "C_LAMBDA", "C_VALUE", "P_VALUE", "ENTROPY_R", "UNROLL_STEP",
                 "REPLAY_MEMORY_LEN", "BUFFER_SIZE", "LEARNER_DEVICE", "REDIS_SERVER", "OPTIM_INFO", "MODEL")
        kw = {k: getattr(C, k) for k in names}
        for k in ("FRAME_DEDUP", "FRAMES_PER_ROLLOUT", "DEDUP_WINDOW", "STAGED_POOL_CODEC",
                  "POOL_BYTES_PER_ROLLOUT"):                                    # optional keys of cfg/impala.json
            if hasattr(C, k):
                kw[k] = getattr(C, k)
        return ImpalaConfig(LOG_W=getattr(C, "LOG_W", None), **kw)


def dedup_geometry(cfg: ImpalaConfig) -> tuple:
    """(pool frames, window) of a FRAME_DEDUP replay: ceil(FRAMES_PER_ROLLOUT * REPLAY_MEMORY_LEN) frames, and
    DEDUP_WINDOW capped at an eighth of them (as apex.dedup_geometry and r2d2.dedup_geometry).  A slot stays live until
    pool - window frames have been stored after it: at the default 24 frames per slot, 21 REPLAY_MEMORY_LEN frames or
    more, above the ~T = 20 new frames per rollout the reference actors send, so the slot ring wraps first.  The window
    only has to reach back two rollouts of the same actor (the bootstrap stack and checkLength's padding)."""
    return R.dedup_pool_geometry(cfg.FRAMES_PER_ROLLOUT, cfg.REPLAY_MEMORY_LEN, cfg.DEDUP_WINDOW)


def pool_bytes(cfg: ImpalaConfig) -> int | None:
    """Bytes of a STAGED_POOL_CODEC store's frame ring (None without STAGED_POOL_CODEC): R.coded_pool_bytes at
    POOL_BYTES_PER_ROLLOUT bytes per slot, by default (F + 1) x 7 072 for dedup_geometry's F frames.  It must hold
    7 072 (W + 2 + 4 (T + 1)) bytes whatever the frames (DESIGN.md §4.23)."""
    if not cfg.STAGED_POOL_CODEC:
        return None
    return R.coded_pool_bytes(cfg.FRAMES_PER_ROLLOUT, cfg.REPLAY_MEMORY_LEN, cfg.POOL_BYTES_PER_ROLLOUT)


def rollout_frames(store):
    """conv_1's frame rows over a rollout store's `state`, row slot * (T + 1) + t being stack t of the slot: the
    field viewed as one stack per row, or a RolloutDedupReplay's plane table."""
    src = store.frame_source("state")
    return src if isinstance(src, R.PlaneFrames) else src.view(-1, 4, 84, 84)


class Replay(ReplayThread):
    """IMPALA/ReplayMemory.py Replay: batch = (s[T+1,B,28224], a[T,B], mu[T,B], r[T,B], done[B]).  run() drains
    `trajectory` (IMPALA/ReplayMemory.py:56-76); the learner never requests an eviction."""

    LIST_KEY = "trajectory"

    def __init__(self, cfg: ImpalaConfig | None = None, connect=None):
        super().__init__(cfg or ImpalaConfig.from_configuration(), connect)
        if self.cfg.FRAME_DEDUP:
            self.store = R.RolloutDedupReplay(self.cfg.REPLAY_MEMORY_LEN, *dedup_geometry(self.cfg),
                                              T=self.cfg.UNROLL_STEP, device=self.device,
                                              pool_bytes=pool_bytes(self.cfg))
        else:
            self.store = R.DeviceReplay(self.cfg.REPLAY_MEMORY_LEN, R.impala_fields(self.cfg.UNROLL_STEP), self.device)
        self._rng = torch.Generator(device=self.device)        # uniform sampling stream (random.sample in the reference)
        self._rng.manual_seed(0x1A9A1A)

    def push_arrays(self, s, a, mu, r, done):
        n = torch.as_tensor(done).numel()
        with self._lock:
            self.store.push([s, a, mu, r, done], torch.ones(n))     # uniform replay: unit priorities

    def push_records(self, blobs) -> None:
        """ReplayMemory.push (baseline/utils.py:305-309) for the actors' pickled rollouts
        (IMPALA/Player.py:183-190): FIFO ring, oldest rollouts overwritten beyond REPLAY_MEMORY_LEN."""
        if not blobs:
            return
        batch = self._wire_decode(blobs)
        if batch is not None:        # decoded on the device (wire.WireIngest)
            self.push_arrays(*[batch[k] for k in ("state", "action", "mu", "reward", "done")])
            return
        import pickle
        from .wire import decode_impala
        self.push_arrays(*decode_impala([pickle.loads(b) for b in blobs], self.cfg.UNROLL_STEP))

    def _wire_ingest(self):
        from .wire import WireIngest
        return WireIngest("impala", self.device, T=self.cfg.UNROLL_STEP)

    def bufferSave(self, m: int = 1):
        """IMPALA/ReplayMemory.py:30-54 with random.sample's no-replacement semantics."""
        B = self.cfg.BATCHSIZE
        with self._lock:
            idx = self.draw(B * m)
            b = self.store.gather(idx)
        for k in range(m):
            sl = slice(k * B, (k + 1) * B)
            self.deque.append((b["state"][sl].transpose(0, 1).contiguous(), b["action"][sl].t().contiguous(),
                               b["mu"][sl].t().contiguous(), b["reward"][sl].t().contiguous(), b["done"][sl]))

    buffer = bufferSave         # what ReplayThread.sample() calls

    def draw(self, n: int) -> torch.Tensor:
        """n distinct slots, uniformly (random.sample over the list of kept rollouts, baseline/utils.py:310-315).
        The kept rollouts are the ring's valid region [head - size, head): slots reserved for an ingest in flight
        are outside it and are never read while they are being overwritten."""
        size, cap, head = self.store._sizes()
        if n > size:
            raise ValueError("Sample larger than population")      # what random.sample raises
        k = torch.randperm(size, device=self.device, generator=self._rng)[:n]
        tail = (head - size) % cap
        return (k + tail) % cap if tail else k

    def __len__(self):
        return len(self.store)


class Learner(CapturedStep):
    def __init__(self, cfg: ImpalaConfig | None = None, connect=None, start_replay: bool = True, memory=None):
        """`memory`: a replay served from another process (replay_server.DeviceReplayClient built with this
        ImpalaConfig, or anything with its surface: sample / memory).  run() then drives sample() -> train() on it;
        with SERVED_FUSED_STEP it steps on the slot `memory.acquire()` binds instead (see _next_step).  fused_step()
        needs the in-process Replay."""
        self.cfg = cfg or ImpalaConfig.from_configuration()
        if memory is not None and self.cfg.SERVED_FUSED_STEP:
            check_served_fused(self.cfg, memory, R.impala_fields(self.cfg.UNROLL_STEP))
        self.device = torch.device(self.cfg.LEARNER_DEVICE)
        self.model = GraphAgent(self.cfg.MODEL).to(self.device)
        self.model.dense_3xtf32 = bool(self.cfg.DENSE_3XTF32) and self.device.type == "cuda"
        self.mOptim = make_optimizer(self.cfg.OPTIM_INFO, self.model.getParameters())
        self._connect = connect
        self._memory = _attach_replay(self, memory, lambda: Replay(self.cfg, connect), connect, start_replay,
                                      wipe=False)
        self.last = {}
        self._graph = self._static = None
        self._bound = None              # _BoundRollouts, built by the first bound step
        self._drawn = None              # _DrawnRollouts, built by the first captured in-process step
        self._bound_warm = 0            # eager warm-up steps on served slots
        self.launches_per_step = None

    @property
    def memory(self):
        return self._memory

    def _stored(self) -> int:
        """Rollouts in the replay: a served memory reports the server's count through `memory`."""
        return len(self._memory.memory) if self._served else len(self._memory)

    def forward(self, state, action):
        """IMPALA/Learner.py:70-83: pi(a|s) of the taken action and V(s)."""
        out = self.model.forward([state])[0]
        A = self.cfg.ACTION_SIZE
        policy = torch.softmax(out[:, :A], dim=-1)
        pi_a = policy.gather(1, action.view(-1, 1).long())[:, 0]
        return pi_a, out[:, -1]

    def train(self, transition, step=0):
        c = self.cfg
        T, B = c.UNROLL_STEP, c.BATCHSIZE
        dev = self.device
        state, action, mu, reward, done = [torch.as_tensor(x).to(dev) for x in transition]
        fused = c.FUSED_CONV1 and state.dtype == torch.uint8 and fused_first_layer(self.model)
        if fused:   # the staged batch is the frame table: rows already are time-major
            frames = state.contiguous().view((T + 1) * B, 4, 84, 84)
            self._train_core(frames, None, action, mu, reward, done, step)
        else:
            self._train_core(state, "staged", action, mu, reward, done, step)

    def fused_step(self, step=0, use_graph=False):
        """One learner step with everything resident: draw B rollouts uniformly without replacement
        (random.sample, baseline/utils.py:310-315), gather only a / mu / r / done (244 B of the 593 KB rollout),
        run conv_1 over the rollouts' (T+1) frames IN PLACE in the replay payload (row = slot * (T+1) + t,
        time-major; with FRAME_DEDUP through the store's plane table, rollout_frames; with STAGED_POOL_CODEC through
        the staged pool the draw's distinct frames are decoded into, _StagedRollouts), V-trace kernel, loss,
        backward, clip + RMSprop.
        `use_graph`: the step as a CUDA graph (_captured_step), its draw one launch of DeviceReplay.uniform_fetch
        before each replay.  -> `last` (for the graph: its static buffers, plus `idx`)."""
        if use_graph:
            return self._captured_step()
        c = self.cfg
        T, B = c.UNROLL_STEP, c.BATCHSIZE
        mem = self._memory
        st = mem.store
        if not hasattr(self, "_small"):
            self._small = st.alloc_batch(B, ("action", "mu", "reward", "done"))
            self._t_idx = torch.arange(T + 1, device=self.device).view(T + 1, 1)
            self._frames = None if self._staged_pool() is not None else rollout_frames(st)
        idx = mem.draw(B)
        b = st.gather(idx, self._small)
        staged = self._staged_pool()
        if staged is not None:
            frames, rows = staged.stage(idx), staged.rows
        else:
            frames, rows = self._frames, time_major_rows(idx, self._t_idx)
        self._train_core(frames, rows, b["action"].t().contiguous(), b["mu"].t().contiguous(),
                         b["reward"].t().contiguous(), b["done"], step)
        return self.last

    def _staged_pool(self) -> "_StagedRollouts | None":
        """The staged frame pool of a STAGED_POOL_CODEC store, built once per learner and shared by the eager and
        captured steps (None for a store conv_1 reads in place)."""
        if not hasattr(self, "_staged"):
            st = self._memory.store
            self._staged = _StagedRollouts(st, self.cfg.BATCHSIZE) if getattr(st, "coded", False) else None
        return self._staged

    def _drawn_state(self) -> "_DrawnRollouts":
        if self._drawn is None:
            self._drawn = _DrawnRollouts(self)
        return self._drawn

    def _captured_step(self):
        """fused_step(use_graph=True): one launch of DeviceReplay.uniform_fetch draws B rollouts into fixed buffers
        (the draw of the served fill, on the replay's device-resident Philox stream), then _train_core runs on them
        with conv_1 reading the frames in place through the fixed frame rows.  The draw reads the host-side size and
        head, so it stays outside the graph.  The first call runs three eager warm-ups, each on its own draw, and
        captures the body on a fourth; every later call is one draw plus graph.replay().  All under the replay's
        lock.  -> `last`: the graph's static buffers, plus `idx`."""
        if self._served:
            raise RuntimeError("fused_step() samples the learner's own replay; a served replay is driven by run()")
        c = self.cfg
        T, B = c.UNROLL_STEP, c.BATCHSIZE
        mem = self._memory
        s = self._drawn_state()
        cur = s.cur

        def draw():
            mem.store.uniform_fetch(B, T, cur)

        def body():
            if s.staged is not None:
                frames, rows = s.staged.stage(cur["idx"]), s.staged.rows
            else:
                frames, rows = s.frames, cur["rows"]
            self._train_core(frames, rows, cur["action"], cur["mu"], cur["reward"], cur["done"], 0)
            self.last["idx"] = cur["idx"]
            return self.last

        def warm_up():
            draw()
            return body()

        # The draw and the replay go to the current stream, as the eager step's draw and gather do, under the lock the
        # replay thread's ingest (Replay.push_arrays) takes: the draw sees the slots committed before it and never
        # those an ingest has reserved, and an ingest enqueued after this call is ordered after the step.
        with mem._lock:
            if self._graph is None:
                self._warm_up(warm_up, 3, s.stream)
                draw()
                self.last = self._eager_or_captured(body, True, s.stream)
            else:
                draw()
                self._graph.replay()
                self.last = self._static
        return self.last

    def _bound_state(self) -> "_BoundRollouts":
        if self._bound is None:
            self._bound = _BoundRollouts(self)
        return self._bound

    def _bound_step(self, use_graph: bool = True):
        """One step on the served rollouts `memory.acquire(cur, frames)` bound (SERVED_FUSED_STEP): _train_core with
        conv_1 and its weight gradient reading the slot's time-major frames through the frame table and a / mu / r /
        done read from the bound buffers.  Warm-up, capture and replay: CapturedStep._served_step.
        -> `last` (for the graph: its static buffers)."""
        s = self._bound_state()
        c = s.cur

        def body():
            self._train_core(s.frames["state"], None, c["action"], c["mu"], c["reward"], c["done"], 0,
                             seq_frames=s.seq_frames)
            return self.last

        self.last = self._served_step(body, use_graph, s.stream)
        return self.last

    def _train_core(self, frames, rows, action, mu, reward, done, step, seq_frames=None):
        """IMPALA/Learner.py:121-235 on a uint8 frame table read in place (`rows`: time-major frame rows, None =
        all rows in order) or, with rows == "staged", on a staged (T+1, B, 28224) batch through PyTorch's first layer.
        The model's first layer is conv_1 or, for a RESCNN2D model, the residual network's stem (R.stem_fused).
        `seq_frames`: with rows None and `frames` a bound ring slot (R.BoundFrames), the same slot's first T * B
        rows, which the grad pass reads (a BoundFrames cannot be sliced)."""
        c = self.cfg
        T, B, A = c.UNROLL_STEP, c.BATCHSIZE, c.ACTION_SIZE
        dev = self.device
        fused = not isinstance(rows, str)
        stem = fused and self.model.first_stem_node() is not None
        with torch.no_grad():
            if stem:
                # one launch: the residual network's stem (conv + max-pool) of all (T+1)*B frame stacks
                if not hasattr(self, "_stem_pack"):
                    self._stem_pack = R.StemPack(dev)
                w1 = getattr(self.model, self.model.first_stem_node()).conv_1.weight
                self._stem_pack.pack(w1)
                p_all, a_all = R.stem_fused(frames, rows, self._stem_pack)
                p_seq, a_seq = p_all[:T * B], a_all[:T * B]
                out_last = self.model.forward_from_stem(p_all[T * B:])[0]
                out_seq = self.model.forward_from_stem(p_seq)[0]
            elif fused:
                # one launch: conv_1 of all (T+1)*B frame stacks, uint8 -> /255 folded in, no fp32 staging
                if not hasattr(self, "_pack1"):
                    self._conv_name, self._pack1 = conv1_packs(self.model, dev, 1)
                w1 = getattr(self.model, self._conv_name).conv_1.weight
                self._pack1.pack(0, w1)
                y_all = R.conv1_fused(frames, rows, self._pack1, relu=False)[0]
                y_seq, y_last = y_all[:T * B], y_all[T * B:]
                out_last = self.model.forward_from_conv1(y_last, False)[0]
                out_seq = self.model.forward_from_conv1(y_seq, False)[0]
            else:
                s = frames.float().div_(255.0).view(T + 1, B, 4, 84, 84)        # :131-140
                last, seq = s[-1], s[:-1].reshape(-1, 4, 84, 84)
                out_last = self.model.forward([last])[0]
                out_seq = self.model.forward([seq])[0]
            boot = (out_last[:, -1] * done.float().view(-1)).contiguous()       # :143
            policy = torch.softmax(out_seq[:, :A], dim=-1)                      # forward(), :70-83
            pi_a = policy.gather(1, action.reshape(-1, 1).long())[:, 0]
            value = out_seq[:, -1]
            vt, adv = R.vtrace(pi_a.view(T, B).contiguous(), mu.float().view(T, B).contiguous(),
                               value.view(T, B).contiguous(), boot, reward.float().view(T, B).contiguous(),
                               c.GAMMA, c.C_LAMBDA, c.C_VALUE, c.P_VALUE)       # :151-215 in one launch
        # calLoss (:95-119): second forward with grad (conv_1's or the stem's output is reused: same weights, same frames)
        if fused:
            if seq_frames is None:
                seq_frames = frames[:T * B] if rows is None else frames
            seq_rows = None if rows is None else rows[:T * B]
        if stem:
            pooled = StemGathered.apply(w1, seq_frames, seq_rows, p_seq, a_seq)
            out = self.model.forward_from_stem(pooled)[0]
        elif fused:
            y = Conv1Gathered.apply(w1, seq_frames, seq_rows, self._pack1, torch.contiguous_format, None, y_seq)
            out = self.model.forward_from_conv1(y, False)[0]
        else:
            out = self.model.forward([seq])[0]
        logp = torch.log_softmax(out[:, :A], dim=-1)
        p = logp.exp()
        entropy = -(p * logp).sum(-1, keepdim=True)
        sel = logp.gather(1, action.reshape(-1, 1).long())
        obj_actor = torch.mean(sel * adv.view(-1, 1) + c.ENTROPY_R * entropy)
        critic = torch.mean((out[:, -1] - vt.view(-1)).pow(2)) / 2
        self.mOptim.zero_grad(set_to_none=False)
        (-obj_actor + critic).backward()                                         # :223-225
        self.step(step)
        self.last = {"objActor": obj_actor.detach(), "criticLoss": critic.detach(), "vtarget": vt, "advantage": adv}

    def step(self, step=0):
        """IMPALA/Learner.py:258-266: clip at 40, RMSprop."""
        self.model.clippingNorm(40)
        self.mOptim.step()

    def state_dict(self):
        return ({k: v.cpu() for k, v in self.model.state_dict().items()},)

    def run(self, max_steps=None):
        """IMPALA/Learner.py:274-297: per step sample -> train, publish `params` (the 1-tuple of the state dict)
        and `Count` EVERY step (:286-287), checkpoint every 100 steps (:290-297).  Publication is asynchronous:
        the weights are snapshot on the learner stream and SET once their D2H copy has landed; if the previous
        snapshot is still in flight this step's is skipped (the actors poll every 400 env steps anyway)."""
        import time
        while self._stored() <= self.cfg.BUFFER_SIZE:
            time.sleep(0.05)
        pub = ParamPublisher(self.model, self._connect, "params", "Count", wrap=lambda sd: (sd,))
        self._publishers, ckpt = publishers(self.model, self.cfg.LOG_W, pub)
        t = 0
        while max_steps is None or t < max_steps:
            if not self._next_step(t):
                time.sleep(0.2)
                continue
            pub.snapshot(t)
            if ckpt is not None and (t + 1) % 100 == 0:
                ckpt.snapshot(t)
            for p in self._publishers:
                p.poll()
            t += 1
        return t

    def _next_step(self, t: int) -> bool:
        """One step of run(): sample() -> train(); or, with SERVED_FUSED_STEP on a served memory, bind the oldest
        filled slot (memory.acquire), run the bound step on it and hand the slot back once the step is enqueued
        (memory.release: conv_1's weight gradient, in backward, is its last reader).  Uniform replay: nothing is
        written back.  -> False when no minibatch is ready (nothing ran)."""
        if self._served and self.cfg.SERVED_FUSED_STEP:
            s = self._bound_state()
            if self._memory.acquire(s.cur, s.frames) is None:
                return False
            self._bound_step()
            self._memory.release()
            return True
        tr = self._memory.sample()
        if tr is False:
            return False
        self.train(tr, t)
        return True


class _BoundRollouts:
    """The buffers a served rollout slot is bound to, built once before the first warm-up, and the stream the bound
    step is warmed up and captured on.  memory.acquire() copies the slot's header, idx, w, action / mu / reward
    (T, B) and done (B,) into `cur` and writes the address of its `state` rows into the one-entry `table`.  The
    server writes the slot time-major (b2rl_serve_fill_uniform), so `state` is conv_1's frame table as it lies:
    (T+1) * B rows in order, no index array.  The grad pass reads its first T * B rows: `seq_frames`, the same table
    entry with fewer rows."""

    def __init__(self, L: "Learner"):
        c, dev = L.cfg, L.device
        T, B = c.UNROLL_STEP, c.BATCHSIZE
        if not fused_first_layer(L.model):
            raise ValueError("SERVED_FUSED_STEP reads the ring slot's frames with the fused conv_1 or stem kernels: "
                             "the model's first node must be the Atari conv_1 or a RESCNN2D stem")
        self.stream = torch.cuda.Stream(dev)
        self.cur = _rollout_buffers(T, B, dev)
        self.cur.update(w=torch.empty(B, dtype=torch.float32, device=dev),
                        header=torch.zeros(2, dtype=torch.int64, device=dev))
        self.table = torch.zeros(1, dtype=torch.int64, device=dev)
        self.frames = {"state": R.BoundFrames(self.table, 0, (T + 1) * B)}
        self.seq_frames = R.BoundFrames(self.table, 0, T * B)


class _DrawnRollouts:
    """The fixed buffers of the captured in-process step (fused_step(use_graph=True)), built once before its first
    warm-up, and the stream it is warmed up and captured on.  DeviceReplay.uniform_fetch draws into `cur`: idx (B,),
    action / mu / reward (T, B), done (B,) and `rows`, the (T+1) * B time-major rows of the drawn rollouts' frames in
    `frames`, the replay's `state` field with one frame stack per row (row = slot * (T+1) + t), or with FRAME_DEDUP
    the store's plane table with the same rows (rollout_frames).  With STAGED_POOL_CODEC the step stages the drawn
    rollouts' frames instead (`staged`), and reads them through the staged pool's fixed rows."""

    def __init__(self, L: "Learner"):
        c, dev = L.cfg, L.device
        T, B = c.UNROLL_STEP, c.BATCHSIZE
        if not fused_first_layer(L.model):
            raise ValueError("fused_step(use_graph=True) reads the replay's frames with the fused conv_1 or stem "
                             "kernels: the model's first node must be the Atari conv_1 or a RESCNN2D stem")
        self.stream = torch.cuda.Stream(dev)
        self.cur = _rollout_buffers(T, B, dev)
        self.staged = L._staged_pool()
        if self.staged is None:
            self.cur["rows"] = torch.empty((T + 1) * B, dtype=torch.int64, device=dev)
            self.frames = rollout_frames(L._memory.store)


class _StagedRollouts:
    """The staged frame pool of a STAGED_POOL_CODEC store (R.RolloutDedupReplay.stage_frames, DESIGN.md §4.23),
    allocated once per learner: B 4 (T + 1) frames and their plane table.  stage(idx) decodes the distinct frames of the
    drawn rollouts into it (one launch, captured with the step) and returns conv_1's frame source; `rows` are its fixed
    time-major rows, row t * B + k = k (T + 1) + t being stack t of draw k."""

    def __init__(self, store, B: int):
        T = store.T
        self.store = store
        self.buffers = store.alloc_staged(B)
        self.rows = time_major_rows(torch.arange(B, device=store.device),
                                    torch.arange(T + 1, device=store.device).view(T + 1, 1))

    def stage(self, idx: torch.Tensor):
        return self.store.stage_frames(idx, self.buffers)


def _rollout_buffers(T: int, B: int, dev) -> dict:
    """A captured step's fixed rollout buffers: action / mu / reward (T, B) and done (B,) with the record's dtypes,
    idx (B,)."""
    f = {x.name: x for x in R.impala_fields(T)}
    cur = {name: torch.empty((T, B), dtype=f[name].dtype, device=dev) for name in ("action", "mu", "reward")}
    cur.update(done=torch.empty(B, dtype=f["done"].dtype, device=dev), idx=torch.empty(B, dtype=torch.int64, device=dev))
    return cur
