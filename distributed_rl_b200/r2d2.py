"""R2D2 learner side with the reference's surface (R2D2/ReplayMemory.py:23-185,
R2D2/Learner.py:39-339): sequences of FIXED_TRAJECTORY steps with a stored LSTM
state live in HBM; burn-in, double-Q n-step targets with value rescaling, the
mixed max/mean sequence priority and dLoss/dQ come from one kernel
(b2rl_r2d2_target) instead of a D2H hop into NumPy fp64 (R2D2/Learner.py:145-181).

SURVEY §8a-note 1: the shipped action slice `action[FIXED_TRAJECTORY-MEM:-1]`
(:111) only runs when MEM == T/2; `[MEM:-1]` (what :120 uses for the rewards)
is used here, identical whenever the reference runs at all.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch

from . import replay as R
from .agent import GraphAgent
from .learner_common import (Conv1Gathered, MemoryView, ReplayThread, StemGathered, TargetNetLearner, _attach_replay,
                             check_served_fused, conv1_packs, fused_first_layer, make_optimizer,
                             require_fused_first_layer, time_major_rows)


def default_r2d2_model() -> dict:
    """cfg/r2d2.json:33-103 (configuration values)."""
    return {
        "module00": {"netCat": "CNN2D", "iSize": 4, "nLayer": 4, "fSize": [8, 4, 3, -1], "nUnit": [32, 64, 64],
                     "padding": [0, 0, 0], "stride": [4, 2, 1], "act": ["relu", "relu", "relu"],
                     "BN": [False] * 4, "linear": True, "input": [0], "prior": 0},
        "module01": {"netCat": "ViewV2", "prevNodeNames": ["module00"], "input": [1], "prior": 1},
        "module02": {"netCat": "LSTMNET", "hiddenSize": 512, "nLayer": 1, "iSize": 3136, "device": "cpu",
                     "FlattenMode": True, "return_hidden": False, "prior": 2, "prevNodeNames": ["module01"]},
        "module03": {"netCat": "MLP", "iSize": 512, "nLayer": 2, "fSize": [512, 6], "act": ["relu", "linear"],
                     "BN": [False] * 3, "prior": 3, "prevNodeNames": ["module02"]},
        "module03_1": {"netCat": "MLP", "iSize": 512, "nLayer": 2, "fSize": [512, 1], "act": ["relu", "linear"],
                       "BN": [False] * 3, "prior": 3, "prevNodeNames": ["module02"]},
        "module04": {"netCat": "Add", "prior": 4, "prevNodeNames": ["module03", "module03_1"]},
        "module04_1": {"netCat": "Mean", "prior": 4, "prevNodeNames": ["module03"]},
        "module05": {"netCat": "Substract", "prior": 5, "prevNodeNames": ["module04", "module04_1"],
                     "output": True},
    }


def resnet_model() -> dict:
    """default_r2d2_model() with the IMPALA paper's residual torso in front of the LSTM, the R2D2 paper's DMLab-30
    agent (R2D2+): module00 is impala.resnet_small_model()'s RESCNN2D node (16, 32, 32 channels, two blocks per
    section, 84 -> 11) and the LSTM takes its 3 872 features; the dueling heads are unchanged.  9 607 744 parameters.
    R2D2Config(MODEL=resnet_model()) trains it; with FUSED_CONV1 its stem reads the sampled sequences' frames in place
    for both networks (R.stem_fused_pair)."""
    from .impala import resnet_small_model
    m = default_r2d2_model()
    m["module00"] = dict(resnet_small_model()["module00"])
    m["module02"]["iSize"] = 3872
    return m


@dataclass
class R2D2Config:
    BATCHSIZE: int = 32
    ACTION_SIZE: int = 6
    ALPHA: float = 0.9
    BETA: float = 0.4
    GAMMA: float = 0.997
    UNROLL_STEP: int = 5
    FIXED_TRAJECTORY: int = 80
    MEM: int = 20
    USE_RESCALING: bool = True
    REPLAY_MEMORY_LEN: int = 10000
    BUFFER_SIZE: int = 1000
    TARGET_FREQUENCY: int = 2500
    LEARNER_DEVICE: str = "cuda:0"
    REDIS_SERVER: str = "localhost"
    LOG_W: str | None = None
    OPTIM_INFO: dict = field(default_factory=lambda: {"name": "adam", "lr": 1e-4, "eps": 0.001})
    MODEL: dict = field(default_factory=default_r2d2_model)
    PAYLOAD_POOL: int = 0        # > 0: the sum-tree has REPLAY_MEMORY_LEN slots but only this many distinct sequences
                                 #      are stored, slot s reading row s % PAYLOAD_POOL (2^20 x 2.26 MB = 2.4 TB
                                 #      does not fit HBM; SURVEY §8d C3).  Benchmark-only; ingest needs 0.
    FUSED_CONV1: bool = True     # conv_1 of every frame through libb2rl's wgmma kernel (gather fused)
    FUSED_HEADS: bool = True     # dueling heads: 3xTF32 wgmma GEMM + fused tail kernels (csrc/gemm.cu, csrc/dueling.cu)
    SERVED_FUSED_STEP: bool = False  # on a served replay (DeviceReplayClient), run() steps a captured step on the
                                     # bound ring slot instead of sample() -> train() -> update()
    FRAME_STRIP: bool = False    # store each sequence's T + 3 distinct frames instead of its T stacks (3.83x fewer
                                 # bytes per sequence at T = 80); conv_1 reads stack t as frames t .. t + 3 in place.
                                 # Only records whose stacks slide (every one R2D2/Player.py sends) can be stored.
    HOST_FRAMES: bool = False    # keep the replay's `state` field (the frames: 99.2 % of a strip sequence's bytes) in
                                 # pinned host memory; the small fields and the sum-tree stay in HBM.  Each step copies
                                 # the sampled sequences' frames over PCIe into a device staging buffer (DESIGN §4.17).
                                 # Replaces PAYLOAD_POOL as the way to a replay larger than HBM, with real ingest.
    FRAME_DEDUP: bool = False    # store every distinct frame once, in a pool of FRAMES_PER_SEQUENCE frames per slot
                                 # (R.StripDedupReplay, DESIGN §4.18): the half-overlapping sequences an actor sends
                                 # share their frames.  Records are frame strips (FRAME_STRIP is set with it), and the
                                 # samples are a strip store's.
    FRAMES_PER_SEQUENCE: float = 48.0
    DEDUP_WINDOW: int = 1 << 14  # a frame is reused only from the last DEDUP_WINDOW frames stored (at most 1/8 of the
                                 # pool, see dedup_geometry)
    HOST_POOL: bool = False      # keep a FRAME_DEDUP store's frame pool in pinned, mapped host memory; the plane table,
                                 # the keys and the sum-tree stay in HBM.  Each step copies the sampled sequences' frames
                                 # over PCIe into a device staging buffer, as HOST_FRAMES does (DESIGN §4.19).
    POOL_CODEC: bool = False     # store a FRAME_DEDUP store's frames losslessly encoded in a ring of bytes in HBM
                                 # (DESIGN §4.21); each step decodes the sampled sequences' frames into a device
                                 # staging buffer, as HOST_POOL copies them.
    POOL_BYTES_PER_SEQUENCE: float | None = None   # POOL_CODEC's ring: this many bytes per slot (see pool_bytes);
                                                   # size it from StripDedupReplay.codec_stats()

    def __post_init__(self):
        if self.HOST_FRAMES and self.PAYLOAD_POOL:
            raise ValueError("HOST_FRAMES stores every sequence's frames in host memory and replaces the PAYLOAD_POOL "
                             "benchmark stand-in: set PAYLOAD_POOL = 0 with HOST_FRAMES")
        if self.HOST_POOL and not self.FRAME_DEDUP:
            raise ValueError("HOST_POOL places the frame pool of a FRAME_DEDUP store: set FRAME_DEDUP with it "
                             "(HOST_FRAMES places a strip or stack store's frames)")
        if self.FRAME_DEDUP and (self.HOST_FRAMES or self.PAYLOAD_POOL):
            raise ValueError("FRAME_DEDUP keeps its frames in a frame pool (in host memory with HOST_POOL) and stores "
                             "every pushed sequence: it takes neither HOST_FRAMES nor PAYLOAD_POOL")
        if self.POOL_CODEC and self.HOST_POOL:
            raise ValueError("POOL_CODEC keeps its coded frame pool in HBM: it does not take HOST_POOL")
        R.check_codec_keys(self, "POOL_CODEC", "POOL_BYTES_PER_SEQUENCE")
        if self.FRAME_DEDUP:
            self.FRAME_STRIP = True

    @staticmethod
    def from_configuration():
        import configuration as C
        names = ("BATCHSIZE", "ACTION_SIZE", "ALPHA", "BETA", "GAMMA", "UNROLL_STEP", "FIXED_TRAJECTORY", "MEM",
                 "USE_RESCALING", "REPLAY_MEMORY_LEN", "BUFFER_SIZE", "TARGET_FREQUENCY", "LEARNER_DEVICE",
                 "REDIS_SERVER", "OPTIM_INFO", "MODEL")
        kw = {k: getattr(C, k) for k in names}
        for k in ("FRAME_DEDUP", "FRAMES_PER_SEQUENCE", "DEDUP_WINDOW", "HOST_POOL", "POOL_CODEC",
                  "POOL_BYTES_PER_SEQUENCE"):                                    # optional keys of cfg/r2d2.json
            if hasattr(C, k):
                kw[k] = getattr(C, k)
        return R2D2Config(LOG_W=getattr(C, "LOG_W", None), FRAME_STRIP=bool(getattr(C, "FRAME_STRIP", False)),
                          HOST_FRAMES=bool(getattr(C, "HOST_FRAMES", False)), **kw)


def dedup_geometry(cfg: R2D2Config) -> tuple:
    """(pool frames, window) of a FRAME_DEDUP replay: ceil(FRAMES_PER_SEQUENCE * REPLAY_MEMORY_LEN) frames, and
    DEDUP_WINDOW capped at an eighth of them (as apex.dedup_geometry).  A slot stays live until pool - window frames
    have been stored after it: at the default 48 frames per slot, 42 REPLAY_MEMORY_LEN frames or more, above the
    ~40 new frames per sequence the reference actors send (T / 2 in mid-episode), so the slot ring wraps first.  The
    window only has to reach back to the same actor's previous sequence."""
    return R.dedup_pool_geometry(cfg.FRAMES_PER_SEQUENCE, cfg.REPLAY_MEMORY_LEN, cfg.DEDUP_WINDOW)


def pool_bytes(cfg: R2D2Config) -> int | None:
    """Bytes of a POOL_CODEC store's frame ring (None without POOL_CODEC): R.coded_pool_bytes at
    POOL_BYTES_PER_SEQUENCE bytes per slot, by default (F + 1) x 7 072 for dedup_geometry's F frames."""
    if not cfg.POOL_CODEC:
        return None
    return R.coded_pool_bytes(cfg.FRAMES_PER_SEQUENCE, cfg.REPLAY_MEMORY_LEN, cfg.POOL_BYTES_PER_SEQUENCE)


class Replay(ReplayThread):
    """R2D2/ReplayMemory.py Replay: batch = [(h0, h1), s, a, r, notdone, w, idx] (:118-120).  The reference's
    update() is unlocked (:48-51); the device handle needs `_lock`."""

    def __init__(self, cfg: R2D2Config | None = None, connect=None):
        super().__init__(cfg or R2D2Config.from_configuration(), connect)
        fields = R.r2d2_config_fields(self.cfg)
        if self.cfg.PAYLOAD_POOL:
            self.store = R.DeviceReplay(self.cfg.REPLAY_MEMORY_LEN, (), self.device)          # priorities only
            self.pool = R.DeviceReplay(self.cfg.PAYLOAD_POOL, fields, self.device)           # the stored sequences
        elif self.cfg.FRAME_DEDUP:
            self.store = self.pool = R.StripDedupReplay(self.cfg.REPLAY_MEMORY_LEN, *dedup_geometry(self.cfg),
                                                        T=self.cfg.FIXED_TRAJECTORY, device=self.device,
                                                        host_pool=self.cfg.HOST_POOL, pool_bytes=pool_bytes(self.cfg))
        else:
            self.store = R.DeviceReplay(self.cfg.REPLAY_MEMORY_LEN, fields, self.device,
                                        host_fields=("state",) if self.cfg.HOST_FRAMES else ())
            self.pool = self.store
        self.memory = MemoryView(self.store, self.cfg.BETA)

    def push_arrays(self, s, a, r, h0, h1, notdone, p):
        """`s`: (n, T, 4, 84, 84) stacks or, with FRAME_STRIP (and so FRAME_DEDUP), (n, T + 3, 84, 84) strips.  With
        FRAME_STRIP, stacks are encoded into strips first (R.encode_strips): a record whose stacks do not slide raises
        ValueError naming it, and nothing of the batch is pushed."""
        if self.cfg.FRAME_STRIP and tuple(s.shape[1:]) != (self.cfg.FIXED_TRAJECTORY + 3, 84, 84):
            s = R.encode_strips(s)
        with self._lock:
            self.store.push([s, a, r, h0, h1, notdone], p)
        self.total_frame += int(torch.as_tensor(p).numel())

    def push_records(self, blobs) -> None:
        """PER.push for the actors' pickled sequences (R2D2/Player.py:312-319) with the indexing of
        R2D2/ReplayMemory.py:70-88: decoded on the device (wire.WireIngest), or on the host when the batch must take
        that path whole (a sequence that does not slide into a strip raises ValueError naming it, nothing pushed)."""
        if not blobs:
            return
        batch = self._wire_decode(blobs)
        if batch is not None:        # decoded on the device (wire.WireIngest), strips already encoded
            self.push_arrays(*[batch[k] for k in ("state", "action", "reward", "h0", "h1", "notdone", "p")])
            return
        import pickle
        from .wire import decode_r2d2
        cols, p = decode_r2d2([pickle.loads(b) for b in blobs], self.cfg.FIXED_TRAJECTORY, strip=self.cfg.FRAME_STRIP)
        self.push_arrays(*cols, p)

    def _wire_ingest(self):
        from .wire import WireIngest
        return WireIngest("r2d2", self.device, T=self.cfg.FIXED_TRAJECTORY, strip=self.cfg.FRAME_STRIP)

    def buffer(self, m: int = 1):
        B = self.cfg.BATCHSIZE
        with self._lock:
            idx, _, w = self.store.sample(B * m, beta=self.cfg.BETA)
            b = self.pool.gather(self.rows_of(idx))
        state = R.as_stacks(b["state"])                     # strips: the zero-copy stack view
        for k in range(m):
            sl = slice(k * B, (k + 1) * B)
            h0 = b["h0"][sl].unsqueeze(0).contiguous()     # (1, B, 512) like torch.cat(..., 1) at :87-88
            h1 = b["h1"][sl].unsqueeze(0).contiguous()
            self.deque.append([(h0, h1), state[sl], b["action"][sl], b["reward"][sl], b["notdone"][sl],
                               w[sl], idx[sl]])

    def rows_of(self, idx: torch.Tensor) -> torch.Tensor:
        """payload row of each sampled slot (identity unless PAYLOAD_POOL)."""
        return idx % self.cfg.PAYLOAD_POOL if self.cfg.PAYLOAD_POOL else idx


class Learner(TargetNetLearner):
    LOG_LINE = ("step:{step} // mean_value:{mean_value:.3f} // norm: {norm:.3f} // REWARD:{reward:.3f} // "
                "NUM_MEMORY:{num_memory} // MAX_WEIGHT:{max_weight:.3f} // TIME:{time_per_step:.5f}")
    PUBLISH_EVERY = 25
    LOG_STATS = ("mean_value", "norm")

    def __init__(self, cfg: R2D2Config | None = None, connect=None, start_replay: bool = True, writer=None,
                 memory=None):
        """`memory`: a replay served from another process (replay_server.DeviceReplayClient or Replay_Server built
        with this R2D2Config, or anything with the `Replay` surface: sample / update / lock / memory).  run() drives
        sample() -> train() -> update() either way; a served memory passes the eviction request on to its server.
        With SERVED_FUSED_STEP, run() over a served memory steps on the slot `memory.acquire()` binds instead (same
        cadence): see _next_step."""
        self.cfg = cfg or R2D2Config.from_configuration()
        if memory is not None and self.cfg.SERVED_FUSED_STEP:
            check_served_fused(self.cfg, memory, R.r2d2_config_fields(self.cfg))
        self.device = torch.device(self.cfg.LEARNER_DEVICE)
        self.model = GraphAgent(self.cfg.MODEL).to(self.device)
        self.target_model = GraphAgent(self.cfg.MODEL).to(self.device)
        for m in (self.model, self.target_model):
            m.dense_3xtf32 = m.fused_dueling_tail = bool(self.cfg.FUSED_HEADS) and self.device.type == "cuda"
        self.optim = make_optimizer(self.cfg.OPTIM_INFO, self.model.getParameters())
        self.connect = connect
        self.memory = _attach_replay(self, memory, lambda: Replay(self.cfg, connect), connect, start_replay, wipe=True)
        self.writer = writer
        self._graph = self._static = None
        self._step_state = None         # _StepState, built by the first captured or bound step
        self._bound_warm = 0            # eager warm-up steps on served slots
        self.launches_per_step = None

    def train(self, transition, t=0):
        c = self.cfg
        T, MEM, B, A = c.FIXED_TRAJECTORY, c.MEM, c.BATCHSIZE, c.ACTION_SIZE
        L = T - MEM
        (h0, h1), state, action, reward, notdone, weight, idx = transition
        dev = self.device
        weight = torch.as_tensor(weight).to(dev, torch.float32)
        h0, h1 = h0.to(dev), h1.to(dev)
        self.model.setCellState((h0, h1))                       # :86-87
        self.target_model.setCellState((h0, h1))
        state = torch.as_tensor(state).to(dev)
        fused = c.FUSED_CONV1 and state.dtype == torch.uint8 and fused_first_layer(self.model)
        if fused:
            strips = R.stacks_strips(state)
            if strips is not None:                              # the stack view of frame strips: read the windows
                frames, pitch = R.strip_windows(strips.contiguous()), T + 3
            else:
                frames, pitch = state.contiguous().view(B * T, 4, 84, 84), T
            q, q_target = self._forward_fused(frames, self._time_major_rows(None, T, B, pitch), T, MEM, B, A)
        else:
            state = state.float() / 255.0                       # :89-90
            sv = state.permute(1, 0, 2, 3, 4).contiguous()      # time-major, :93
            burn = sv[:MEM].reshape(-1, 4, 84, 84)
            window = sv[MEM:].reshape(-1, 4, 84, 84)
            with torch.no_grad():                               # burn-in, :99-104
                shape = torch.tensor([MEM, B, -1])
                self.model.forward([burn, shape])
                self.target_model.forward([burn, shape])
                self.model.detachCellState()
                self.target_model.detachCellState()
            shape = torch.tensor([L, B, -1])
            q = self.model.forward([window, shape])[0].view(L, B, A)              # :121
            with torch.no_grad():
                q_target = self.target_model.forward([window, shape])[0].view(L, B, A)   # :132
        out, info = self._learn(q, q_target, action, reward, notdone, weight)
        info["mean_value"] = out["scalars"][1]
        info["loss"] = out["scalars"][0]
        return info, out["prio"], idx

    def _learn(self, q, q_target, action, reward, notdone, weight):
        """The step after the forward passes (R2D2/Learner.py:110-215): the window's actions / rewards, target and
        priority kernel, backward, then step().  `action`, `reward`: (B, T); `notdone`, `weight`: (B,).
        -> (the target kernel's outputs, step()'s info)"""
        c, dev = self.cfg, self.device
        MEM = c.MEM
        act = torch.as_tensor(action).to(dev, torch.int64).t()[MEM:-1].contiguous()      # (L-1, B)
        rew = torch.as_tensor(reward).to(dev, torch.float32).t()[MEM:-1].contiguous()
        nd = torch.as_tensor(notdone).to(dev, torch.float32).contiguous()
        out = R.r2d2_target(q.detach().contiguous(), q_target.contiguous(), act, rew, nd, weight,
                            c.UNROLL_STEP, c.GAMMA, c.ALPHA, c.USE_RESCALING)
        q.backward(out["grad_q"])                               # == loss.backward(), :189-192
        return out, self.step()

    def _time_major_rows(self, seq_rows, T, B, pitch):
        """Frame-table rows of the (t, b) frames in time-major order: row = seq_row[b] * pitch + t (pitch T for
        stacks, T + 3 for the windows of frame strips; seq_rows None: the batch itself is the table, sequence b's
        rows start at b * pitch)."""
        if not hasattr(self, "_t_idx"):
            self._t_idx = torch.arange(T, device=self.device).view(T, 1)
            self._b_idx = torch.arange(B, device=self.device)
        return time_major_rows(self._b_idx if seq_rows is None else seq_rows, self._t_idx, pitch)

    def _forward_fused(self, frames, tm_rows, T, MEM, B, A):
        """The forward passes with conv_1 on the tensor cores, reading `frames` (a uint8 (rows, 4, 84, 84) table:
        the staged batch or the replay payload itself, its stacks or the windows of its strips) IN PLACE: the (b, t) ->
        time-major reordering and the uint8 -> /255 conversion are folded into the kernel's gather (`tm_rows`).  A
        RESCNN2D model runs its stem instead (_forward_stem)."""
        if self.model.first_stem_node() is not None:
            return self._forward_stem(frames, tm_rows, T, MEM, B, A)
        dev = self.device
        if not hasattr(self, "_pack2"):
            self._conv_name, self._pack2, self._pack1 = conv1_packs(self.model, dev, 2, 1)
        w_on = getattr(self.model, self._conv_name).conv_1.weight
        w_tg = getattr(self.target_model, self._conv_name).conv_1.weight
        self._pack2.pack(0, w_on); self._pack2.pack(1, w_tg); self._pack1.pack(0, w_on)
        rows_burn, rows_win = tm_rows[:MEM * B], tm_rows[MEM * B:]
        L = T - MEM
        with torch.no_grad():                                   # burn-in, :99-104
            y_on, y_tg = R.conv1_fused(frames, rows_burn, self._pack2, relu=True)
            shape = torch.tensor([MEM, B, -1])
            self.model.forward_from_conv1(y_on, True, [shape])
            self.target_model.forward_from_conv1(y_tg, True, [shape])
            self.model.detachCellState()
            self.target_model.detachCellState()
            y_on_w, y_tg_w = R.conv1_fused(frames, rows_win, self._pack2, relu=False)
        shape = torch.tensor([L, B, -1])
        mf = torch.contiguous_format
        y = Conv1Gathered.apply(w_on, frames, rows_win, self._pack1, mf, None, y_on_w)
        q = self.model.forward_from_conv1(y, False, [shape])[0].view(L, B, A)             # :121
        with torch.no_grad():
            q_target = self.target_model.forward_from_conv1(torch.relu(y_tg_w), True, [shape])[0].view(L, B, A)
        return q, q_target

    def _forward_stem(self, frames, tm_rows, T, MEM, B, A):
        """_forward_fused for a RESCNN2D model: the residual network's stem (3x3 conv + max-pool) of both networks in
        one launch per pass (R.stem_fused_pair), reading `frames` in place through `tm_rows`.  The online net's grad
        pass takes the window's pooled output through StemGathered, whose backward runs the stem's weight-gradient
        kernel over the same rows; only that pass needs the argmax."""
        if not hasattr(self, "_stem_packs"):
            self._stem_packs = R.stem_pack_pair(self.device)
        name = self.model.first_stem_node()
        w_on = getattr(self.model, name).conv_1.weight
        pack_on, pack_tg = self._stem_packs
        pack_on.pack(w_on)
        pack_tg.pack(getattr(self.target_model, name).conv_1.weight)
        rows_burn, rows_win = tm_rows[:MEM * B], tm_rows[MEM * B:]
        L = T - MEM
        with torch.no_grad():                                   # burn-in, :99-104
            p_on, p_tg, _ = R.stem_fused_pair(frames, rows_burn, pack_on, pack_tg, argmax=False)
            shape = torch.tensor([MEM, B, -1])
            self.model.forward_from_stem(p_on, [shape])
            self.target_model.forward_from_stem(p_tg, [shape])
            self.model.detachCellState()
            self.target_model.detachCellState()
            p_on_w, p_tg_w, a_on_w = R.stem_fused_pair(frames, rows_win, pack_on, pack_tg)
        shape = torch.tensor([L, B, -1])
        pooled = StemGathered.apply(w_on, frames, rows_win, p_on_w, a_on_w)
        q = self.model.forward_from_stem(pooled, [shape])[0].view(L, B, A)              # :121
        with torch.no_grad():
            q_target = self.target_model.forward_from_stem(p_tg_w, [shape])[0].view(L, B, A)   # :132
        return q, q_target

    def fused_step(self, use_graph: bool = False):
        """One learner step with everything resident: sample B sequence slots + IS weights from the sum-tree,
        gather only the small per-sequence fields (a, r, h0, h1, notdone: 5 KB of the 2.26 MB), run conv_1 over the
        sequences' frames IN PLACE in the replay payload (row = slot_row * T + t), target / priority kernel,
        backward, clip + Adam, priority write-back.  No host round trip (R2D2/Learner.py:235-274 in one call).
        `use_graph`: the first call runs three eager warm-ups and captures the step as a CUDA graph (under the
        replay's lock, so that no ingest work lands in the capture); every later call replays it.  The draw reads
        the tree's device-resident size and Philox counter, so each replay draws a new minibatch.
        With FRAME_DEDUP conv_1 reads each stack's four frames from the frame pool through the slots' plane table
        (R.StripDedupReplay.frame_source), with the rows of a strip store.  With HOST_FRAMES or HOST_POOL the frames
        are not in HBM: the same gather launch sequence also copies the sampled sequences' `state` rows (with
        HOST_POOL their strips, assembled from the host pool) from host memory into a fixed device staging buffer,
        and conv_1 reads that buffer with the rows train() uses on a staged batch (row = b * pitch + t).  With
        POOL_CODEC the frames are encoded: the same gather decodes the sampled strips into that staging buffer."""
        if self._graph is not None:
            self._graph.replay()
            return self._static
        if self._served:
            raise RuntimeError("fused_step() samples the learner's own replay; a served replay is driven by run()")
        c = self.cfg
        T, MEM, B, A = c.FIXED_TRAJECTORY, c.MEM, c.BATCHSIZE, c.ACTION_SIZE
        mem = self.memory
        st, pool = mem.store, mem.pool
        staged = c.HOST_FRAMES or c.HOST_POOL or c.POOL_CODEC   # the frames are in host memory, or encoded
        if not hasattr(self, "_small"):
            self._small = pool.alloc_batch(B, ("action", "reward", "h0", "h1", "notdone"))
            if staged:
                self._small.update(pool.alloc_batch(B, ("state",)))    # the staging buffer: B sequences' frames
                buf = self._small["state"]
                self._frames = R.strip_windows(buf) if c.FRAME_STRIP else buf.view(-1, 4, 84, 84)
                self._pitch = T + 3 if c.FRAME_STRIP else T
            elif c.FRAME_DEDUP:                                         # the windows through the plane table
                self._frames, self._pitch = pool.frame_source("state"), T + 3
            elif c.FRAME_STRIP:
                self._frames, self._pitch = R.strip_windows(pool.field_view("state")), T + 3
            else:
                self._frames, self._pitch = pool.field_view("state").view(-1, 4, 84, 84), T

        def body():
            idx, _, w = st.sample(B, beta=c.BETA, want_prob=False)
            rows = mem.rows_of(idx)
            b = pool.gather(rows, self._small)
            h0, h1 = b["h0"].unsqueeze(0), b["h1"].unsqueeze(0)
            self.model.setCellState((h0, h1))
            self.target_model.setCellState((h0, h1))
            seq_rows = None if staged else rows                 # staged: sequence b's frames start at row b * pitch
            q, q_target = self._forward_fused(self._frames, self._time_major_rows(seq_rows, T, B, self._pitch), T, MEM,
                                              B, A)
            out, info = self._learn(q, q_target, b["action"], b["reward"], b["notdone"], w)
            st.update(idx, out["prio"])
            return {"scalars": out["scalars"], "p_norm": info["p_norm"], "prio": out["prio"], "idx": idx}

        if not use_graph:
            return body()
        stream = self._state().stream
        with mem._lock:
            self._warm_up(body, 3, stream)
            return self._eager_or_captured(body, True, stream)

    def _state(self) -> "_StepState":
        if self._step_state is None:
            self._step_state = _StepState(self)
        return self._step_state

    def _bound_step(self, use_graph: bool = True):
        """One step on the served minibatch `memory.acquire(cur, frames)` bound (SERVED_FUSED_STEP): fused_step's
        body with the draw, the small-field gather and the tree update replaced by the bound buffers; conv_1 of the
        burn-in, of the window and its weight gradient read the slot's frames through the frame table.  The
        priorities leave through memory.update() after the step.  Warm-up, capture and replay:
        CapturedStep._served_step."""
        s = self._state()
        c, cur = self.cfg, s.cur
        T, MEM, B, A = c.FIXED_TRAJECTORY, c.MEM, c.BATCHSIZE, c.ACTION_SIZE
        h0, h1 = cur["h0"].unsqueeze(0), cur["h1"].unsqueeze(0)

        def body():
            self.model.setCellState((h0, h1))
            self.target_model.setCellState((h0, h1))
            q, q_target = self._forward_fused(s.frames["state"], s.rows, T, MEM, B, A)
            out, info = self._learn(q, q_target, cur["action"], cur["reward"], cur["notdone"], cur["w"])
            return {"scalars": out["scalars"], "p_norm": info["p_norm"], "prio": out["prio"], "idx": cur["idx"]}

        return self._served_step(body, use_graph, s.stream)

    def step(self):
        """R2D2/Learner.py:200-215: norm, clip at 40, Adam."""
        params = self.model.getParameters()
        grads = [p.grad for p in params if p.grad is not None]
        p_norm = torch.stack(torch._foreach_norm(grads, 2)).sum().sqrt()
        torch.nn.utils.clip_grad_norm_(params, 40, foreach=True)
        self.optim.step()
        self.optim.zero_grad(set_to_none=False)
        return {"p_norm": p_norm}

    def _next_step(self, step: int, log_every: int):
        """One iteration of run() (R2D2/Learner.py:240-274): sample -> train -> the write-back cadence.  With
        SERVED_FUSED_STEP on a served memory, the oldest filled slot is bound (memory.acquire), the bound step runs
        on it and the slot is handed back once the step is enqueued (memory.release: conv_1's weight gradient, in
        backward, is its last reader); then the write-back.
        -> {mean(Q), norm} as a device tensor, or None when no minibatch is ready."""
        if self._served and self.cfg.SERVED_FUSED_STEP:
            s = self._state()
            if self.memory.acquire(s.cur, s.frames) is None:
                return None
            out = self._bound_step()
            self.memory.release()
            self._write_back(step, log_every, out["idx"], out["prio"])
            return torch.stack([out["scalars"][1].reshape(()), out["p_norm"].reshape(())])
        batch = self.memory.sample()
        if batch is False:
            return None
        info, prio, idx = self.train(batch)
        self._write_back(step, log_every, idx, prio)
        return torch.stack([info["mean_value"].reshape(()), info["p_norm"].reshape(())])


class _StepState:
    """What a captured R2D2 step keeps from one step to the next, built once before its first warm-up: the stream it
    is warmed up and captured on and, on a served memory, the buffers a ring slot is bound to.  memory.acquire()
    copies the slot's header, idx, w, action (B, T), reward (B, T), h0, h1 (B, 512) and notdone (B,) into `cur` and
    writes the address of its `state` rows into the one-entry `table`.  The slot's `state` is batch-major
    (B, T, 4, 84, 84), so frame (b, t) is row b * T + t from that address (with FRAME_STRIP, (B, T + 3, 84, 84):
    window b * (T + 3) + t, rows 7 056 bytes apart), and `rows` (the time-major order the burn-in and the window
    read, split at MEM * B by _forward_fused) stays the same for every slot."""

    def __init__(self, L: "Learner"):
        c, dev = L.cfg, L.device
        T, B = c.FIXED_TRAJECTORY, c.BATCHSIZE
        require_fused_first_layer(L.model, "SERVED_FUSED_STEP" if L._served else "fused_step(use_graph=True)")
        self.stream = torch.cuda.Stream(dev)
        self.cur = self.frames = self.rows = None
        if L._served:
            self.cur = dict(R.alloc_rows(R.r2d2_config_fields(c), B, dev, ("action", "reward", "h0", "h1", "notdone")),
                            idx=torch.empty(B, dtype=torch.int64, device=dev),
                            w=torch.empty(B, dtype=torch.float32, device=dev),
                            header=torch.zeros(2, dtype=torch.int64, device=dev))
            self.table = torch.zeros(1, dtype=torch.int64, device=dev)
            pitch, rows, stride = R.sequence_rows(B, T, c.FRAME_STRIP)
            self.frames = {"state": R.BoundFrames(self.table, 0, rows, stride)}
            self.rows = L._time_major_rows(None, T, B, pitch)
