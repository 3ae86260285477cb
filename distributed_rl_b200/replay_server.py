"""Stand-alone replay mode (SURVEY.md §8 f4): `ReplayServer` (APE_X/ReplayServer.py:20-160,
R2D2/ReplayServer.py:20-175) owns the prioritized replay in ITS OWN process / GPU and serves pre-assembled minibatches
over the reference's Redis protocol; `Replay_Server` (APE_X/ReplayMemory.py:170-257, R2D2/ReplayMemory.py:187-274) is
the learner-side consumer with the `Replay` surface (`sample()`, `update()`, `start()`).  Every server and client
serves the record kind of its config: Ape-X transitions (`ApexConfig`), R2D2 sequences (`R2D2Config`) or, on the
device ring only, IMPALA rollouts (`ImpalaConfig`), see `KINDS`.  The reference has no IMPALA replay server, so the
Redis-protocol pair refuses an ImpalaConfig.

Keys (the reference's): list `experience` (actors -> server), list `BATCH` on the push connection (server ->
learner: pickled `[s, a, r, s', done, w, idx]` or `[(h0, h1), s, a, r, notdone, w, idx]`), list `update` (learner ->
server: pickled `(idx list, priorities)`), flags `FLAG_BATCH` (enough data to serve), `FLAG_ENOUGH` (learner has more
than 32 (Ape-X) / 18 (R2D2) batches queued), `FLAG_REMOVE` (learner asks for `remove_to_fit`).

What is GPU-native here is the server's store: sampling, IS weights, gather and priority write-back are the HBM
kernels of libb2rl (one sample launch + one TMA gather per served group of minibatches, applied updates in stream
order); the transport stays the reference's pickled Redis lists — this mode exists so that a deployment which
runs the reference's replay out of process keeps working, not as the fast path (the in-process `Replay` is).
Lists are drained atomically (`wire.drain`), see wire.py.

`DeviceReplayServer` / `DeviceReplayClient` are the GPU-native transport beside them: minibatches are drawn and
assembled by ONE kernel (`b2rl_serve_fill`) straight into a ring of device slots that the learner maps through CUDA
IPC, and priorities come back through update slots of the same ring; no minibatch or priority touches the host.
Redis carries only small descriptors and the handles (DESIGN.md §4.15):

  key   SERVE_RING     ring IPC handle + layout + the server's events (filled[k], applied[j])   server -> learner
  key   SERVE_CLIENT   the learner's events (released[k], written[j])                          learner -> server
  key   SERVE_STATS    (len(replay), max IS weight), for `memory`                              server -> learner
  key   SERVE_DETACHED the learner has unmapped the ring: the server may free it               learner -> server
  list  BATCH_SLOT     (k, seq, n): minibatch slot k holds fill `seq`                          server -> learner
  list  RELEASE_SLOT   (k, seq): the learner's copy out of slot k is enqueued                  learner -> server
  list  UPDATE_SLOT    (j, seq, n): update slot j holds n (idx, priority) pairs                learner -> server
  list  UPDATE_DONE    (j, seq): the server's tree update of slot j is enqueued                server -> learner

Event invariant: an interprocess event is re-recorded only after the host-level handshake for its slot has
completed, and a peer's stream waits on it only after reading the descriptor posted behind the record.  So every
`cudaStreamWaitEvent` waits on the intended record, and no kernel ever waits for the other process: a missing peer
leaves slots unserved, it cannot hang a GPU.

Shutdown: the learner closes its client first (unmap, then SERVE_DETACHED); the server frees the ring only after
that key appears.  A learner that attached with `apex.Learner(connect=..., memory=client)` or
`r2d2.Learner(connect=..., memory=client)` keeps SERVER_KEYS out of its start-up wipe of stale keys
(`impala.Learner` wipes no keys).

IMPALA rollouts are unprioritized: the server fills a slot with `b2rl_serve_fill_uniform` (B distinct rollouts drawn
uniformly from the valid region, written time-major so that `state` is conv_1's frame table as it lies in the slot),
publishes a max IS weight of 0 and never receives update slots."""
from __future__ import annotations

import ctypes as C
import pickle
import threading
import time
from collections import deque
from dataclasses import dataclass
from typing import Callable

import numpy as np
import torch

from . import _lib, wire
from . import replay as R
from ._lib import check
from . import apex, impala, r2d2
from .apex import ApexConfig
from .impala import ImpalaConfig
from .learner_common import Stoppable, _index_tensor
from .r2d2 import R2D2Config


@dataclass(frozen=True)
class RecordKind:
    """What the servers and clients need to know about the records they serve."""
    name: str
    replay: type                    # the ingest Replay: decoder of the actors' records + the store
    fields: Callable                # cfg -> the store's fields
    batch: Callable                 # (gathered fields, IS weights, indices) -> the learner's minibatch list
    host: Callable | None           # (field name, CPU tensor) -> what a pickled `BATCH` blob carries
    m: int                          # minibatches per ReplayServer.buffer()
    enough: int                     # Replay_Server raises FLAG_ENOUGH above this many queued minibatches
    list_key: str = "experience"    # the actors' Redis list the server drains
    steps: Callable | None = None   # cfg -> T for a uniform, time-major kind (IMPALA); None: prioritized, batch-major

    @property
    def prioritized(self) -> bool:
        return self.steps is None


def _apex_batch(b, w, idx):
    """APE_X/ReplayServer.py:95-114: [s, a, r, s', done, w, idx]."""
    return [b["state"], b["action"], b["reward"], b["next_state"], b["done"], w, idx]


def _r2d2_batch(b, w, idx):
    """R2D2/ReplayMemory.py:74-120 (r2d2.Replay.buffer): [(h0, h1), s, a, r, notdone, w, idx], h0 / h1 (1, B, 512),
    s (B, T, 4, 84, 84): the stack view of frame strips."""
    return [(b["h0"].unsqueeze(0), b["h1"].unsqueeze(0)), R.as_stacks(b["state"]), b["action"], b["reward"],
            b["notdone"], w, idx]


def _r2d2_host(name, t):
    """A pickled R2D2 `BATCH` keeps the reference's format: h0 / h1 stay torch (:100-101), s is the (B, T, 4, 84, 84)
    stack array, materialised here from frame strips."""
    if name in ("h0", "h1"):
        return t
    return np.ascontiguousarray(R.as_stacks(t).numpy()) if name == "state" else t.numpy()


def _impala_batch(b, w, idx):
    """IMPALA/ReplayMemory.py:30-54 (impala.Replay.bufferSave): (s, a, mu, r, done), s (T+1, B, 28224) time-major."""
    return (b["state"], b["action"], b["mu"], b["reward"], b["done"])


KINDS = {
    "apex": RecordKind("apex", apex.Replay, lambda cfg: R.APEX_FIELDS, _apex_batch,
                       lambda name, t: t.numpy().astype(bool) if name == "done" else t.numpy(),
                       m=32, enough=32),                      # APE_X/ReplayServer.py:66, APE_X/ReplayMemory.py:232
    "r2d2": RecordKind("r2d2", r2d2.Replay, R.r2d2_config_fields, _r2d2_batch, _r2d2_host,
                       m=8, enough=18),                       # R2D2/ReplayServer.py:66, R2D2/ReplayMemory.py:249
    "impala": RecordKind("impala", impala.Replay, lambda cfg: R.impala_fields(cfg.UNROLL_STEP), _impala_batch,
                         None, m=1, enough=0, list_key="trajectory",           # IMPALA/ReplayMemory.py:56-76
                         steps=lambda cfg: cfg.UNROLL_STEP),
}


def record_kind(cfg) -> RecordKind:
    """The kind a config describes: R2D2Config -> sequences, ImpalaConfig -> rollouts, anything else (ApexConfig)
    -> transitions."""
    if isinstance(cfg, R2D2Config):
        return KINDS["r2d2"]
    return KINDS["impala" if isinstance(cfg, ImpalaConfig) else "apex"]


def _redis_protocol_kind(cfg) -> None:
    """The Redis-protocol pair serves the reference's two replay servers (Ape-X, R2D2) and nothing else."""
    if cfg is not None and not record_kind(cfg).prioritized:
        raise ValueError(f"the Redis-protocol replay server has no {record_kind(cfg).name} mode (the reference has no "
                         "IMPALA replay server): serve it with DeviceReplayServer / DeviceReplayClient")


class _StandaloneServer(Stoppable):
    """What the two stand-alone servers share (APE_X/ReplayServer.py:20-160, R2D2/ReplayServer.py:20-175): the
    ingest of the actors' records (`experience`, IMPALA's `trajectory`) into the store, FLAG_BATCH once the store
    holds more than BUFFER_SIZE records, and eviction on FLAG_REMOVE.  `cfg`: ApexConfig (the default, from
    `configuration`), R2D2Config or ImpalaConfig."""

    def __init__(self, cfg: ApexConfig | R2D2Config | ImpalaConfig | None, connect):
        super().__init__()
        self.cfg = cfg or ApexConfig.from_configuration()
        if getattr(self.cfg, "PAYLOAD_POOL", 0):
            raise ValueError("a replay server needs a store that ingests records; PAYLOAD_POOL is a benchmark store "
                             "without ingest (set PAYLOAD_POOL = 0)")
        self.kind = record_kind(self.cfg)
        self.device = torch.device(self.cfg.LEARNER_DEVICE)
        self._ingest = self.kind.replay(self.cfg, connect=None)   # never started: record decoder + staging + store
        self.store = self._ingest.store
        self.connect = connect
        self.FLAG_BATCH = False
        self.total_transition = 0

    def _ingest_experience(self) -> list:
        """The top of serve_once(): raise FLAG_BATCH, then push the drained records of the kind's list. -> the
        records."""
        if len(self.store) > self.cfg.BUFFER_SIZE and not self.FLAG_BATCH:
            self.FLAG_BATCH = True
            self.connect.set("FLAG_BATCH", pickle.dumps(True))
        data = wire.drain(self.connect, self.kind.list_key)
        if data:
            self._ingest.push_records(data)
            self.total_transition += len(data)
        return data

    def _evict_on_request(self) -> None:
        """A full store honours the learner's FLAG_REMOVE: evict down to REPLAY_MEMORY_LEN, clear the flag."""
        if len(self.store) >= self.cfg.REPLAY_MEMORY_LEN:
            cond = self.connect.get("FLAG_REMOVE")
            if cond is not None and pickle.loads(cond):
                over = len(self.store) - self.cfg.REPLAY_MEMORY_LEN
                if over > 0:
                    self.store.evict(over)
                self.connect.set("FLAG_REMOVE", pickle.dumps(False))


class ReplayServer(_StandaloneServer):
    def __init__(self, cfg: ApexConfig | R2D2Config | None = None, connect=None, connect_push=None,
                 m: int | None = None):
        _redis_protocol_kind(cfg)
        super().__init__(cfg, connect)
        self.connect_push = connect_push if connect_push is not None else connect
        self.m = self.kind.m if m is None else m   # minibatches per buffer() (the reference: Ape-X 32, R2D2 8; :66)
        self.FLAG_REMOVE = False
        if self.connect is not None:
            self.connect.set("FLAG_BATCH", pickle.dumps(False))           # :39

    def update(self) -> int:
        """:41-63 — apply the learner's queued priority write-backs."""
        data = wire.drain(self.connect, "update")
        if not data:
            return 0
        idx_list, vals_list = [], []
        for d in data:
            idx, vals = pickle.loads(d)
            idx_list += [int(i) for i in idx]
            vals_list.append(np.asarray(vals, np.float32))
        self.store.update(torch.as_tensor(np.asarray(idx_list, np.int64)).to(self.device),
                          torch.as_tensor(np.concatenate(vals_list, 0)).to(self.device))
        return len(idx_list)

    def buffer(self) -> int:
        """APE_X/ReplayServer.py:65-114, R2D2/ReplayServer.py:65-136 — sample BATCHSIZE * m, IS weights, assemble m
        minibatches, RPUSH them to `BATCH`, each once.  R2D2 minibatch k is sequences kB .. kB + B - 1, batch-major
        (state (B, T, 4, 84, 84)), the layout r2d2.Replay.buffer hands its learner (DESIGN.md §2: the reference's
        time-major vsplit and its second RPUSH of every blob are not reproduced)."""
        B, m = self.cfg.BATCHSIZE, self.m
        idx, _, w = self.store.sample(B * m, beta=self.cfg.BETA)
        b = {name: t.cpu() for name, t in self.store.gather(idx).items()}
        w, idx = w.cpu(), idx.cpu()
        blobs = []
        for k in range(m):
            sl = slice(k * B, (k + 1) * B)
            host = {name: self.kind.host(name, t[sl]) for name, t in b.items()}
            blobs.append(pickle.dumps(self.kind.batch(host, w[sl], idx[sl])))
        return self.connect_push.rpush("BATCH", *blobs)

    def serve_once(self) -> dict:
        """One iteration of run() (:116-160)."""
        data = self._ingest_experience()
        pushed = self.buffer() if data and len(self.store) > self.cfg.BUFFER_SIZE else 0
        applied = self.update()
        self._evict_on_request()
        return {"ingested": len(data), "batches_queued": pushed, "updates_applied": applied}

    def run(self):
        while not self._stop_evt.is_set():
            st = self.serve_once()
            if st["batches_queued"] > 100:
                time.sleep(1)                   # the learner is behind: :143-144
            elif not st["ingested"]:
                time.sleep(0.002)


class Replay_Server(Stoppable, threading.Thread):
    """Learner-side consumer of a ReplayServer: same surface as `Replay` (sample / update / start / lock).  Every
    `BATCH` blob is queued once and unpickled once, by sample() (R2D2/ReplayMemory.py:244-246 queues each blob a
    second time, already unpickled, which its sample() then fails to unpickle; DESIGN.md §2)."""

    def __init__(self, cfg: ApexConfig | R2D2Config | None = None, connect=None, connect_push=None):
        _redis_protocol_kind(cfg)
        super().__init__(daemon=True)
        self.cfg = cfg or ApexConfig.from_configuration()
        self.kind = record_kind(self.cfg)
        self.connect, self.connect_push = connect, connect_push if connect_push is not None else connect
        self._lock = threading.Lock()
        self.deque, self.idx, self.vals = [], [], []
        self.lock = False

    def update(self, idx, vals) -> None:
        """:188-190 — queue; flushed to the server's `update` list beyond 1000 entries."""
        with self._lock:
            self.idx += [int(i) for i in idx]
            self.vals.append(np.asarray(vals.detach().cpu() if torch.is_tensor(vals) else vals, np.float32))

    def poll_once(self) -> None:
        data = wire.drain(self.connect_push, "BATCH")
        if data:
            with self._lock:
                self.deque += data
        self.connect.set("FLAG_ENOUGH", pickle.dumps(len(self.deque) > self.kind.enough))   # :232-239
        if self.lock:                                                              # eviction request -> the server's flag
            self.connect.set("FLAG_REMOVE", pickle.dumps(True))
            self.lock = False
        with self._lock:
            if len(self.idx) > 1000:                                               # :241-249
                self.connect.rpush("update", pickle.dumps((self.idx[:], np.concatenate(self.vals, 0))))
                self.idx.clear(); self.vals.clear()

    def run(self):
        while not self._stop_evt.is_set():
            self.poll_once()
            time.sleep(0.001)

    def sample(self):
        with self._lock:
            if not self.deque:
                return False
            blob = self.deque.pop(0)
        return pickle.loads(blob)


# ---- device serve ring ----------------------------------------------------------------------------------------------
RING_KEY, CLIENT_KEY, STATS_KEY, DETACH_KEY = "SERVE_RING", "SERVE_CLIENT", "SERVE_STATS", "SERVE_DETACHED"
BATCH_SLOT, RELEASE_SLOT, UPDATE_SLOT, UPDATE_DONE = "BATCH_SLOT", "RELEASE_SLOT", "UPDATE_SLOT", "UPDATE_DONE"
# What a running DeviceReplayServer reads or owns: a learner attached to it must not wipe these at start-up
# (the server resets its own keys when it starts).
SERVER_KEYS = (RING_KEY, CLIENT_KEY, STATS_KEY, DETACH_KEY, BATCH_SLOT, RELEASE_SLOT, UPDATE_SLOT, UPDATE_DONE,
               "experience", "FLAG_BATCH", "FLAG_REMOVE")


def serve_layout(batch: int, slots: int, field_bytes) -> _lib.ServeLayout:
    """The ring geometry for a replay whose fields have these row sizes (b2rl_serve_layout_init; no CUDA call)."""
    L = _lib.ServeLayout()
    fb = (C.c_int64 * _lib.MAX_FIELDS)(*[int(b) for b in field_bytes])
    check(_lib.load().b2rl_serve_layout_init(int(batch), int(slots), len(field_bytes), fb, C.byref(L)))
    return L


def bind_targets(batch: int, fields, out: dict, frames: dict):
    """The per-field arguments of b2rl_serve_bind for a slot of `batch` records: (copy destinations, frame table
    entries), one pointer per field, null for a field that is neither copied nor bound.  A copied field's buffer holds
    exactly its `batch` rows.  A bound frame field's BoundFrames must cover exactly the FRAME_STACK_BYTES rows, its
    row_stride apart, that fit in the slot's batch * field_bytes: conv_1 reads no further than the slot.  For frame
    stacks that is batch times field_bytes / FRAME_STACK_BYTES (Ape-X one per record, an R2D2 sequence T, an IMPALA
    rollout T + 1); for the windows of R2D2 frame strips, batch * (T + 3) - 3."""
    fo, to = (C.c_void_p * _lib.MAX_FIELDS)(), (C.c_void_p * _lib.MAX_FIELDS)()
    for i, f in enumerate(fields):
        if f.name in out:
            t = out[f.name]
            assert t.is_contiguous() and t.numel() * t.element_size() == batch * f.nbytes, f.name
            fo[i] = t.data_ptr()
        elif f.name in frames:
            bf = frames[f.name]
            span = batch * f.nbytes - R.FRAME_STACK_BYTES
            if span < 0 or bf.rows != span // bf.row_stride + 1:
                raise ValueError(f"field {f.name!r} holds {f.nbytes / R.FRAME_STACK_BYTES:g} frame stacks per record: "
                                 f"a slot of {batch} records has {max(span // bf.row_stride + 1, 0)} frame rows "
                                 f"{bf.row_stride} bytes apart, not the {bf.rows} of its BoundFrames")
            to[i] = frames[f.name].entry_ptr()
    return fo, to


class ServeRing:
    """The ring allocation as seen by this process: created for a DeviceReplay (the server owns it) or mapped from
    an exported IPC handle (the learner)."""

    def __init__(self, handle: C.c_void_p, device: torch.device, owned: bool):
        self.lib = _lib.load()
        self._h, self.device, self.owned = handle, device, owned
        self.layout = _lib.ServeLayout()
        check(self.lib.b2rl_serve_ring_layout(self._h, C.byref(self.layout)))

    @classmethod
    def create(cls, store: R.DeviceReplay, batch: int, slots: int) -> "ServeRing":
        h = C.c_void_p()
        check(_lib.load().b2rl_serve_ring_create(store._h, int(batch), int(slots), C.byref(h)))
        return cls(h, store.device, True)

    @classmethod
    def open(cls, handle: bytes, layout: bytes, device) -> "ServeRing":
        device = torch.device(device)
        L = _lib.ServeLayout.from_buffer_copy(layout)
        buf = C.create_string_buffer(bytes(handle), _lib.IPC_HANDLE_BYTES)
        h = C.c_void_p()
        with torch.cuda.device(device):
            torch.zeros(1, device=device)          # the primary context the mapping lives in
            check(_lib.load().b2rl_serve_ring_open(buf, C.byref(L), device.index, C.byref(h)))
        return cls(h, device, False)

    def export(self) -> bytes:
        buf = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
        check(self.lib.b2rl_serve_ring_export(self._h, buf))
        return buf.raw

    def layout_bytes(self) -> bytes:
        return bytes(self.layout)

    def slot_ptrs(self, k: int):
        """-> (minibatch slot pointers {header, idx, w, field 0, ...}, update slot pointers {header, idx, prio})."""
        b, u = (C.c_void_p * (3 + _lib.MAX_FIELDS))(), (C.c_void_p * 3)()
        check(self.lib.b2rl_serve_slot_ptrs(self._h, int(k), b, u))
        return list(b)[:3 + self.layout.n_fields], list(u)

    def fill(self, store: R.DeviceReplay, k: int, seq: int, beta: float, max_w: torch.Tensor | None = None) -> None:
        check(self.lib.b2rl_serve_fill(store._h, self._h, int(k), int(seq), float(beta),
                                       None if max_w is None else max_w.data_ptr(), store._st()))

    def fill_uniform(self, store: R.DeviceReplay, k: int, seq: int, steps: int) -> None:
        """B distinct records drawn uniformly from the store's valid region, time-major over `steps` (IMPALA's T)."""
        check(self.lib.b2rl_serve_fill_uniform(store._h, self._h, int(k), int(seq), int(steps), store._st()))

    def take(self, k: int, dst: torch.Tensor, stream) -> None:
        assert dst.is_contiguous() and dst.numel() * dst.element_size() >= self.layout.slot_bytes
        check(self.lib.b2rl_serve_take(self._h, int(k), dst.data_ptr(), stream.cuda_stream))

    def bind(self, base: int, fields, out: dict, frames: dict, stream) -> None:
        """b2rl_serve_bind: the filled slot at device address `base` (a mapped slot or a local copy of one) -> the
        step's fixed buffers: out["header"] (int64[2]), out["idx"], out["w"] and every field named in `out` are
        copied; every field named in `frames` (name -> R.BoundFrames) gets the address of its rows in the slot."""
        L = self.layout
        fo, to = bind_targets(L.batch, fields, out, frames)
        check(self.lib.b2rl_serve_bind(base, C.byref(L), L.batch, out["header"].data_ptr(), out["idx"].data_ptr(),
                                       out["w"].data_ptr(), fo, to, stream.cuda_stream))

    def put_update(self, j: int, seq: int, idx: torch.Tensor, prio: torch.Tensor, stream) -> None:
        check(self.lib.b2rl_serve_put_update(self._h, int(j), int(seq), idx.data_ptr(), prio.data_ptr(), idx.numel(),
                                             stream.cuda_stream))

    def close(self) -> None:
        if getattr(self, "_h", None):
            (self.lib.b2rl_serve_ring_destroy if self.owned else self.lib.b2rl_serve_ring_close)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ServerSlots:
    """The server's half of the host-level handshake (no CUDA here: the device work is passed in).
    A minibatch slot is free, or out (filled and announced, not yet released by the learner)."""

    def __init__(self, connect, slots: int, batch: int):
        self.connect, self.batch = connect, batch
        self.free = list(range(slots))
        self.out = {}                 # slot -> seq of the fill the learner has not released yet
        self.seq = 0

    def collect_releases(self, wait) -> int:
        """Drain RELEASE_SLOT; `wait(k)` makes the server stream wait on released[k] (recorded by the learner before
        it posted the descriptor) before slot k can be refilled."""
        got = [pickle.loads(d) for d in wire.drain(self.connect, RELEASE_SLOT)]
        for k, seq in got:
            if self.out.get(k) != seq:
                raise RuntimeError(f"release of slot {k} (seq {seq}) that the server did not hand out")
            wait(k)
            del self.out[k]
            self.free.append(k)
        return len(got)

    def apply_updates(self, apply) -> int:
        """Drain UPDATE_SLOT; `apply(j, n)` waits on written[j], applies the slot to the tree and records
        applied[j]; then UPDATE_DONE hands the slots back.  -> number of priorities applied."""
        got = [pickle.loads(d) for d in wire.drain(self.connect, UPDATE_SLOT)]
        for j, _, n in got:
            apply(j, n)
        if got:
            self.connect.rpush(UPDATE_DONE, *[pickle.dumps((j, seq)) for j, seq, _ in got])
        return sum(n for _, _, n in got)

    def fill_free(self, fill) -> int:
        """`fill(k, seq)` fills every free slot and records filled[k]; then the descriptors go out, in fill order."""
        blobs = []
        while self.free:
            k = self.free.pop(0)
            self.seq += 1
            fill(k, self.seq)
            self.out[k] = self.seq
            blobs.append(pickle.dumps((k, self.seq, self.batch)))
        if blobs:
            self.connect.rpush(BATCH_SLOT, *blobs)
        return len(blobs)


class ClientSlots:
    """The learner's half of the handshake (no CUDA here).  Thread-safe: a polling thread may call poll()."""

    def __init__(self, connect, slots: int):
        self.connect = connect
        self.ready = deque()          # (k, seq, n) announced by the server, not yet copied out
        self.upd_free = list(range(slots))
        self.upd_seq = 0
        self._mu = threading.Lock()

    def poll(self) -> None:
        pipe = self.connect.pipeline()
        for key in (BATCH_SLOT, UPDATE_DONE):
            pipe.lrange(key, 0, -1)
            pipe.delete(key)
        r = pipe.execute()
        filled, done = r[0] or [], r[2] or []
        with self._mu:
            self.ready.extend(pickle.loads(d) for d in filled)
            self.upd_free.extend(pickle.loads(d)[0] for d in done)

    def acquire(self):
        """The oldest filled slot, held by the learner until release(k, seq).  -> (k, seq, n), or None when nothing
        is filled."""
        with self._mu:
            return self.ready.popleft() if self.ready else None

    def release(self, k: int, seq: int) -> None:
        """RELEASE_SLOT hands slot k back (the caller has recorded released[k] behind the slot's last reader)."""
        self.connect.rpush(RELEASE_SLOT, pickle.dumps((k, seq)))

    def take(self, copy):
        """The oldest filled slot: `copy(k)` waits on filled[k], copies the slot out and records released[k]; then
        RELEASE_SLOT hands it back.  -> (k, seq, n), or None when nothing is filled."""
        desc = self.acquire()
        if desc is None:
            return None
        copy(desc[0])
        self.release(*desc[:2])
        return desc

    def put_update(self, write, n: int) -> bool:
        """A free update slot j: `write(j, seq)` waits on applied[j], writes the slot and records written[j]; then
        UPDATE_SLOT announces it.  False when every update slot is still with the server."""
        with self._mu:
            if not self.upd_free:
                return False
            j = self.upd_free.pop(0)
            self.upd_seq += 1
            seq = self.upd_seq
        write(j, seq)
        self.connect.rpush(UPDATE_SLOT, pickle.dumps((j, seq, n)))
        return True


def _ipc_events(device: torch.device, n: int):
    """n interprocess events on `device` and their IPC handles (torch creates an event lazily, on the current
    device: the handles are taken inside the device guard)."""
    with torch.cuda.device(device):
        ev = [torch.cuda.Event(interprocess=True) for _ in range(n)]
        return ev, [e.ipc_handle() for e in ev]


class DeviceReplayServer(_StandaloneServer):
    """The stand-alone replay server over a device ring (APE_X/ReplayServer.py:20-160): the same `experience` ingest,
    eviction on FLAG_REMOVE and FLAG_BATCH as `ReplayServer`, but each served minibatch is one `b2rl_serve_fill`
    launch into a ring slot the learner maps through CUDA IPC.  Keeps up to `slots` filled minibatches ahead of the
    learner and applies arriving update slots in stream order.  Run it in its own process (CUDA IPC cannot map a
    handle into the process that exported it)."""

    STATS_EVERY = 0.1             # seconds between SERVE_STATS refreshes (each costs a device sync)

    def __init__(self, cfg: ApexConfig | R2D2Config | ImpalaConfig | None = None, connect=None, slots: int = 4):
        super().__init__(cfg, connect)
        self.device = self.store.device
        self.ring = ServeRing.create(self.store, self.cfg.BATCHSIZE, slots)
        self.slots = ServerSlots(connect, slots, self.cfg.BATCHSIZE)
        (self.filled, filled_h), (self.applied, applied_h) = _ipc_events(self.device, slots), _ipc_events(self.device, slots)
        self.released = self.written = None                # the learner's events, once it has attached
        self._upd = [self.ring.slot_ptrs(j)[1] for j in range(slots)]
        self._stats_t = 0.0
        connect.delete(BATCH_SLOT, RELEASE_SLOT, UPDATE_SLOT, UPDATE_DONE, CLIENT_KEY, STATS_KEY, DETACH_KEY)
        connect.set("FLAG_BATCH", pickle.dumps(False))
        connect.set(RING_KEY, pickle.dumps({
            "handle": self.ring.export(), "layout": self.ring.layout_bytes(), "device": self.device.index,
            "filled": filled_h, "applied": applied_h}))

    def _stream(self):
        return torch.cuda.current_stream(self.device)

    def _peer_events(self):
        """The learner's released / written events (SERVE_CLIENT is set before the learner posts any descriptor)."""
        if self.released is None:
            blob = self.connect.get(CLIENT_KEY)
            if blob is None:
                raise RuntimeError("a descriptor arrived before the learner published its events")
            info = pickle.loads(blob)
            dev = torch.device("cuda", info["device"])
            self.released = [torch.cuda.Event.from_ipc_handle(dev, h) for h in info["released"]]
            self.written = [torch.cuda.Event.from_ipc_handle(dev, h) for h in info["written"]]
        return self.released, self.written

    def _wait_released(self, k: int) -> None:
        self._stream().wait_event(self._peer_events()[0][k])

    def _apply(self, j: int, n: int) -> None:
        st = self._stream()
        st.wait_event(self._peer_events()[1][j])
        _, idx, prio = self._upd[j]
        check(self.store.lib.b2rl_tree_update(self.store._h, idx, prio, int(n), st.cuda_stream))
        self.applied[j].record(st)

    def _fill(self, k: int, seq: int) -> None:
        if self.kind.prioritized:
            self.ring.fill(self.store, k, seq, self.cfg.BETA)
        else:
            self.ring.fill_uniform(self.store, k, seq, self.kind.steps(self.cfg))
        self.filled[k].record(self._stream())

    def _can_fill(self) -> bool:
        """More than BUFFER_SIZE records; a draw without replacement also needs at least B of them."""
        n = len(self.store)
        return n > self.cfg.BUFFER_SIZE and (self.kind.prioritized or n >= self.cfg.BATCHSIZE)

    def _publish_stats(self, force: bool) -> None:
        now = time.time()
        if force or now - self._stats_t > self.STATS_EVERY:
            prio = self.kind.prioritized and len(self.store)
            mw = float(self.store.stats(self.cfg.BETA)[2].item()) if prio else 0.0
            self.connect.set(STATS_KEY, pickle.dumps((len(self.store), mw)))
            self._stats_t = now

    def serve_once(self) -> dict:
        """One iteration of run(): ingest, take back released slots, apply update slots, refill free slots, evict."""
        data = self._ingest_experience()
        released = self.slots.collect_releases(self._wait_released)
        applied = self.slots.apply_updates(self._apply)
        filled = self.slots.fill_free(self._fill) if self._can_fill() else 0
        self._evict_on_request()
        self._publish_stats(bool(data))
        return {"ingested": len(data), "filled": filled, "released": released, "updates_applied": applied}

    def run(self):
        while not self._stop_evt.is_set():
            st = self.serve_once()
            if not (st["ingested"] or st["filled"] or st["released"] or st["updates_applied"]):
                time.sleep(0.0005)

    def close(self, timeout: float = 60.0) -> bool:
        """Free the ring once the learner has unmapped it.  If a learner attached, wait (up to `timeout` s) for its
        SERVE_DETACHED, which DeviceReplayClient.close() sets after unmapping.  Without it the ring is NOT freed —
        a learner may still be copying out of a slot — and is released with this process.  -> True when freed."""
        torch.cuda.synchronize(self.device)
        if self.released is not None or self.connect.get(CLIENT_KEY) is not None:
            t0 = time.time()
            while self.connect.get(DETACH_KEY) is None:
                if time.time() - t0 > timeout:
                    self.ring._h = None          # left mapped: freed with the process, never under a reader
                    return False
                time.sleep(0.01)
        self.ring.close()
        return True


class ServedMemory:
    """`Replay.memory` of a DeviceReplayClient: len() and .max_weight as the server last published them."""

    def __init__(self, connect):
        self._connect = connect

    def _stats(self):
        blob = self._connect.get(STATS_KEY)
        return pickle.loads(blob) if blob is not None else (0, 0.0)

    def __len__(self):
        return int(self._stats()[0])

    @property
    def max_weight(self) -> float:
        return float(self._stats()[1])


class DeviceReplayClient(Stoppable, threading.Thread):
    """Learner-side consumer of a DeviceReplayServer with the `Replay` surface (start / stop / sample / update / lock /
    memory; APE_X/ReplayMemory.py:170-257).  sample() returns `[s, a, r, s', done, w, idx]` as CUDA tensors on the
    learner's device, copied out of the ring (a peer copy when the server is on another GPU); with an R2D2Config,
    `[(h0, h1), s, a, r, notdone, w, idx]` as r2d2.Replay.sample returns it; with an ImpalaConfig,
    `(s, a, mu, r, done)` time-major as impala.Replay.sample returns it (`last_idx` holds the rollouts' slots)."""

    KEEP_KEYS = SERVER_KEYS       # what apex/r2d2.Learner(connect=..., memory=this) leaves in place at start-up

    def __init__(self, cfg: ApexConfig | R2D2Config | ImpalaConfig | None = None, connect=None,
                 timeout: float = 60.0):
        super().__init__(daemon=True)
        self.cfg = cfg or ApexConfig.from_configuration()
        self.kind = record_kind(self.cfg)
        self.device = torch.device(self.cfg.LEARNER_DEVICE)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.connect = connect
        self.lock = False
        t0 = time.time()
        while (blob := connect.get(RING_KEY)) is None:
            if time.time() - t0 > timeout:
                raise TimeoutError(f"no replay server published {RING_KEY} within {timeout} s")
            time.sleep(0.01)
        info = pickle.loads(blob)
        self.ring = ServeRing.open(info["handle"], info["layout"], self.device)
        L = self.ring.layout
        self.fields = self.kind.fields(self.cfg)
        if [L.field_bytes[i] for i in range(L.n_fields)] != [f.nbytes for f in self.fields]:
            raise RuntimeError(f"the server's ring does not carry the {self.kind.name} record fields of this config")
        srv = torch.device("cuda", info["device"])
        self.server_device = srv
        self.filled =[torch.cuda.Event.from_ipc_handle(srv, h) for h in info["filled"]]
        self.applied = [torch.cuda.Event.from_ipc_handle(srv, h) for h in info["applied"]]
        (self.released, released_h), (self.written, written_h) = _ipc_events(self.device, L.slots), \
            _ipc_events(self.device, L.slots)
        connect.set(CLIENT_KEY, pickle.dumps({"device": self.device.index, "released": released_h,
                                              "written": written_h}))
        self.slots = ClientSlots(connect, L.slots)
        self.memory = ServedMemory(connect)
        self._pending = deque()      # priority write-backs waiting for a free update slot
        self.last_served = None      # descriptor (k, seq, n) of the last served slot
        self.last_header = None      # its header {seq, n} as copied out: a device int64[2]
        self.last_idx = None         # its replay slots: a device int64[B]
        self._held = None            # (k, seq) of the slot acquire() bound in place, until release()
        self._stage = None           # acquire() with the server on another GPU: the learner-local slot copy

    def _stream(self):
        return torch.cuda.current_stream(self.device)

    def poll_once(self) -> None:
        self.slots.poll()
        if self.lock:                                   # eviction request -> the server's flag
            self.connect.set("FLAG_REMOVE", pickle.dumps(True))
            self.lock = False

    def run(self):
        while not self._stop_evt.is_set():
            self.poll_once()
            time.sleep(0.0005)

    def _views(self, buf: torch.Tensor):
        L, B = self.ring.layout, self.ring.layout.batch

        def view(off, nbytes, dtype, shape):
            return buf[off:off + nbytes].view(dtype).view(shape)

        def shape(f):            # a time-major slot: step t of record k at row t * B + k; scalars stay (B,)
            if self.kind.prioritized or not f.shape:
                return (B,) + tuple(f.shape)
            return (f.shape[0], B) + tuple(f.shape[1:])
        out = {f.name: view(L.field_off[i], B * f.nbytes, f.dtype, shape(f)) for i, f in enumerate(self.fields)}
        return (view(0, 16, torch.int64, (2,)), view(L.idx_off, 8 * B, torch.int64, (B,)),
                view(L.w_off, 4 * B, torch.float32, (B,)), out)

    def _next_filled(self):
        """The oldest filled slot, held by the learner until it is released, with the current stream made to wait on
        its filled[k].  Polls first while the eviction request is pending or nothing is known to be filled.
        -> (descriptor (k, seq, n), stream), or None when nothing is filled."""
        if self.lock or not self.slots.ready:
            self.poll_once()
        desc = self.slots.acquire()
        if desc is None:
            return None
        cur = self._stream()
        cur.wait_event(self.filled[desc[0]])
        return desc, cur

    def sample(self):
        """Replay_Server.sample (APE_X/ReplayMemory.py:251-257, R2D2/ReplayMemory.py:266-274): the oldest filled
        slot, copied into fresh learner-local memory on the current stream; False when nothing is filled."""
        got = self._next_filled()
        if got is None:
            return False
        desc, cur = got
        k, seq, _ = desc
        buf = torch.empty(self.ring.layout.slot_bytes, dtype=torch.uint8, device=self.device)
        self.ring.take(k, buf, cur)
        self.released[k].record(cur)
        self.slots.release(k, seq)
        header, idx, w, b = self._views(buf)
        self.last_served, self.last_header, self.last_idx = desc, header, idx
        return self.kind.batch(b, w, idx)

    def acquire(self, out: dict, frames: dict):
        """sample() for a captured learner step (SERVED_FUSED_STEP of apex, r2d2 or impala.Learner): the oldest filled
        slot is bound
        to the step's fixed buffers (ServeRing.bind) on the current stream, behind filled[k]; nothing is allocated.
        `out`: header (int64[2]), idx, w and the fields to copy; `frames`: field name -> R.BoundFrames whose table
        entry receives the address of that field's rows.  With the server on this GPU the slot itself is bound and
        stays with the learner until release().  With the server on another GPU the slot is copied once into a
        persistent learner-local buffer and released at once; that buffer is bound.  -> the descriptor (k, seq, n),
        or None when nothing is filled."""
        got = self._next_filled()
        if got is None:
            return None
        desc, cur = got
        k, seq, _ = desc
        if self.server_device == self.device:
            base = self.ring.slot_ptrs(k)[0][0]
            self._held = (k, seq)
        else:
            if self._stage is None:
                self._stage = torch.empty(self.ring.layout.slot_bytes, dtype=torch.uint8, device=self.device)
            self.ring.take(k, self._stage, cur)
            self.released[k].record(cur)
            self.slots.release(k, seq)
            base = self._stage.data_ptr()
        self.ring.bind(base, self.fields, out, frames, cur)
        self.last_served = desc
        return desc

    def release(self) -> None:
        """Hand back the slot acquire() bound in place: released[k] is recorded on the current stream, so call it
        once the step that reads the slot is enqueued (conv_1's weight gradient, in backward, reads it last).  A slot
        that was copied to the learner's GPU has already been released."""
        if self._held is None:
            return
        k, seq = self._held
        self._held = None
        self.released[k].record(self._stream())
        self.slots.release(k, seq)

    def update(self, idx, vals) -> None:
        """Replay_Server.update (APE_X/ReplayMemory.py:188-190): the write-back goes to free update slots of the
        ring (at most B pairs each) and is applied by the server in stream order.  `idx`: a tensor, an array, or a
        list of ints or 0-d tensors.  An unprioritized kind (IMPALA) has no write-back."""
        if not self.kind.prioritized:
            raise TypeError(f"the {self.kind.name} replay is uniform: it has no priorities to write back")
        idx = _index_tensor(idx).to(device=self.device, dtype=torch.int64).reshape(-1).contiguous()
        vals = torch.as_tensor(vals).to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
        assert idx.numel() == vals.numel()
        B = self.ring.layout.batch
        new = 0
        for a in range(0, idx.numel(), B):
            self._pending.append((idx[a:a + B], vals[a:a + B]))
            new += 1
        self._flush_updates()
        # Whatever still waits for an update slot is copied now, on the stream: the caller's tensors may be a captured
        # step's static outputs, which its next replay overwrites.
        for j in range(max(len(self._pending) - new, 0), len(self._pending)):
            i, v = self._pending[j]
            self._pending[j] = (i.clone(), v.clone())

    def _flush_updates(self) -> None:
        cur = self._stream()
        while self._pending:
            i, v = self._pending[0]

            def write(j, seq):
                cur.wait_event(self.applied[j])        # the server's tree update has read the slot's last contents
                self.ring.put_update(j, seq, i, v, cur)
                self.written[j].record(cur)
            if not self.slots.put_update(write, i.numel()):
                self.slots.poll()
                if not self.slots.put_update(write, i.numel()):
                    return                              # every update slot is with the server: retried next time
            self._pending.popleft()

    def close(self) -> None:
        """Unmap the ring, then tell the server (SERVE_DETACHED) that it may free it."""
        torch.cuda.synchronize(self.device)
        self.ring.close()
        self.connect.set(DETACH_KEY, pickle.dumps(True))
