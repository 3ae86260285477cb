"""DeviceReplay — one HBM-resident replay shard (payload SoA + fp64 sum-tree).

Thin, typed wrapper over the C ABI (include/b2rl.h).  All heavy lifting happens
in the CUDA kernels of libb2rl.so; this file only marshals torch tensors'
device pointers and the current CUDA stream.  It is the object the reference-
facing mirrors (per.py: PER / PrioritizedMemory, apex.py: Replay) are built on.
"""
from __future__ import annotations

import ctypes as C
import math
import warnings
from dataclasses import dataclass
from typing import Sequence

import numpy as np
import torch

from . import _lib, hostmem
from ._lib import ReplayDesc, check

FRAME_STACK_BYTES = 4 * 84 * 84  # one (4,84,84) uint8 observation, 28 224 B
FRAME_BYTES = 84 * 84            # one 84x84 uint8 frame, 7 056 B: the row stride of a frame strip's windows


@dataclass(frozen=True)
class Field:
    name: str
    dtype: torch.dtype
    shape: tuple  # per-slot shape

    @property
    def nbytes(self) -> int:
        n = 1
        for s in self.shape:
            n *= int(s)
        return n * torch.empty((), dtype=self.dtype).element_size()


# Record layouts of the three learners (SURVEY.md §8a / §3.4).
APEX_FIELDS = (  # [s, a, R_n, s', done, prio]  APE_X/Player.py:252-261
    Field("state", torch.uint8, (4, 84, 84)),
    Field("next_state", torch.uint8, (4, 84, 84)),
    Field("action", torch.int32, ()),
    Field("reward", torch.float32, ()),
    Field("done", torch.uint8, ()),
)


# The frame-deduplicated Ape-X store (ApexConfig.FRAME_DEDUP, DESIGN.md §4.16): per slot 8 int32 pool ids, planes 0-3
# of s then planes 0-3 of s', into a library-owned ring of 84x84 frames; the scalar fields are APEX_FIELDS' own.
APEX_DEDUP_FIELDS = (Field("planes", torch.int32, (8,)),) + APEX_FIELDS[2:]
DEDUP_HASH_MASK = (1 << 63) - 1     # every key bit; a test passes 0 to make every frame collide


def r2d2_fields(T: int = 80, hidden: int = 512, strip: bool = False):
    """[(h0,h1), (s,a,r) x T, done, prio]  R2D2/ReplayMemory.py:70-88.  `strip`: `state` holds the sequence's T + 3
    distinct frames (T + 3, 84, 84) instead of its T stacks (T, 4, 84, 84); stack t is frames t .. t + 3."""
    return (
        Field("state", torch.uint8, (T + 3, 84, 84) if strip else (T, 4, 84, 84)),
        Field("action", torch.int32, (T,)),
        Field("reward", torch.float32, (T,)),
        Field("h0", torch.float32, (hidden,)),
        Field("h1", torch.float32, (hidden,)),
        Field("notdone", torch.float32, ()),
    )


def r2d2_config_fields(cfg):
    """The R2D2 record fields of an R2D2Config: FIXED_TRAJECTORY steps, frame strips when FRAME_STRIP is set."""
    return r2d2_fields(cfg.FIXED_TRAJECTORY, strip=bool(getattr(cfg, "FRAME_STRIP", False)))


def R2D2_DEDUP_FIELDS(T: int = 80, hidden: int = 512):
    """The slot of the frame-deduplicated R2D2 store (R2D2Config.FRAME_DEDUP, DESIGN.md §4.18): `planes`, the T + 3
    int32 pool ids of the sequence's frame strip (frame j of the strip is pool frame planes[j]), then the small fields
    of r2d2_fields."""
    return (Field("planes", torch.int32, (T + 3,)),) + r2d2_fields(T, hidden, strip=True)[1:]


# ---- R2D2 frame strips: a sequence of T stacks stored as its T + 3 distinct frames ----------------------------------
# Every R2D2 record slides: R2D2/Player.py:38-63 stacks the last four frames of one episode, so stack t + 1 is stack t
# shifted by one frame (s[t+1][:3] == s[t][1:]).  Frames t .. t + 3 of a strip are stack t, and stack t is the
# FRAME_STACK_BYTES that start at byte t * FRAME_BYTES of the strip: conv_1 reads it in place as one row of a view
# whose rows are FRAME_BYTES apart.
def sequence_rows(n_seq: int, T: int, strip: bool) -> tuple:
    """conv_1's frame rows over `n_seq` consecutive sequences of T steps -> (row pitch per sequence, rows, row stride
    in bytes).  Stacks: T rows per sequence, n_seq * T rows of FRAME_STACK_BYTES.  Strips: T + 3 rows per sequence
    (the last three windows of a strip straddle into the next one and are never read), n_seq * (T + 3) - 3 rows, the
    last of which ends at the end of the last strip."""
    if strip:
        return T + 3, n_seq * (T + 3) - 3, FRAME_BYTES
    return T, n_seq * T, FRAME_STACK_BYTES


def strip_windows(strips: torch.Tensor) -> torch.Tensor:
    """The window view of contiguous uint8 strips (n_seq, T + 3, 84, 84): a (n_seq * (T + 3) - 3, 4, 84, 84) view
    with strides (7056, 7056, 84, 1), whose row s * (T + 3) + t is stack t of sequence s.  Zero-copy."""
    assert strips.dtype == torch.uint8 and strips.dim() == 4 and strips.shape[2:] == (84, 84) and strips.is_contiguous()
    _, rows, _ = sequence_rows(strips.shape[0], strips.shape[1] - 3, True)
    return strips.as_strided((rows, 4, 84, 84), (FRAME_BYTES, FRAME_BYTES, 84, 1))


def strip_stacks(strips: torch.Tensor) -> torch.Tensor:
    """The stack view of uint8 strips (B, T + 3, 84, 84) whose inner three dimensions are contiguous: a zero-copy
    (B, T, 4, 84, 84) view whose values are the sequences' stacks."""
    assert strips.dtype == torch.uint8 and strips.dim() == 4 and strips.shape[2:] == (84, 84) and strips[0].is_contiguous()
    B, T = strips.shape[0], strips.shape[1] - 3
    return strips.as_strided((B, T, 4, 84, 84), (strips.stride(0), FRAME_BYTES, FRAME_BYTES, 84, 1))


def stacks_strips(stacks: torch.Tensor) -> torch.Tensor | None:
    """The strips (B, T + 3, 84, 84) under a stack view made by strip_stacks, or None when `stacks` is not one."""
    if stacks.dim() != 5 or stacks.stride()[1:] != (FRAME_BYTES, FRAME_BYTES, 84, 1):
        return None
    B, T = stacks.shape[0], stacks.shape[1]
    return stacks.as_strided((B, T + 3, 84, 84), (stacks.stride(0), FRAME_BYTES, 84, 1))


def as_stacks(state: torch.Tensor) -> torch.Tensor:
    """R2D2 `state` rows as the learner reads them, (B, T, 4, 84, 84): strips through their stack view, stacks as
    they are."""
    return strip_stacks(state) if state.ndim == 4 else state


def encode_strip(stacks, out: np.ndarray, record: int = 0) -> None:
    """One record's T stacks (an iterable of (4, 84, 84) uint8 arrays, e.g. a (T, 4, 84, 84) array) -> its strip
    `out` (T + 3, 84, 84): out[0:4] = s_0, out[3 + t] = s_t[3], after checking s_t[:3] == out[t:t+3].  A stack that
    does not slide raises ValueError naming `record` (its position in the batch) and the step."""
    T = out.shape[0] - 3
    t = -1
    for t, st in enumerate(stacks):
        if t >= T:
            raise ValueError(f"record {record}: more than {T} stacks")
        st = np.asarray(st, np.uint8).reshape(4, 84, 84)
        if t == 0:
            out[0:3] = st[:3]
        elif not np.array_equal(st[:3], out[t:t + 3]):
            raise ValueError(f"record {record}: stack {t} is not stack {t - 1} shifted by one frame, so the sequence "
                             "cannot be stored as a frame strip (FRAME_STRIP)")
        out[3 + t] = st[3]
    if t != T - 1:
        raise ValueError(f"record {record}: {t + 1} stacks, not {T}")


def encode_strips(stacks) -> np.ndarray:
    """(n, T, 4, 84, 84) uint8 stacks -> (n, T + 3, 84, 84) strips (encode_strip per record).  Every record is
    checked before anything is returned, so a caller that pushes the result pushes all of the batch or none of it."""
    stacks = stacks.cpu().numpy() if torch.is_tensor(stacks) else np.asarray(stacks)
    n, T = stacks.shape[:2]
    out = np.empty((n, T + 3, 84, 84), np.uint8)
    for i in range(n):
        encode_strip(stacks[i], out[i], i)
    return out


def impala_fields(T: int = 20):
    """(s[T+1], a[T], mu[T], r[T], done)  IMPALA/ReplayMemory.py:34-43."""
    return (
        Field("state", torch.uint8, (T + 1, 4 * 84 * 84)),
        Field("action", torch.int32, (T,)),
        Field("mu", torch.float32, (T,)),
        Field("reward", torch.float32, (T,)),
        Field("done", torch.float32, ()),
    )


def IMPALA_DEDUP_FIELDS(T: int = 20):
    """The slot of the frame-deduplicated IMPALA store (ImpalaConfig.FRAME_DEDUP, DESIGN.md §4.20): `planes`, the
    4 (T + 1) int32 pool ids of the rollout's T + 1 frame stacks (frame c of stack t is pool frame planes[4 t + c]),
    then the small fields of impala_fields."""
    return (Field("planes", torch.int32, (4 * (T + 1),)),) + impala_fields(T)[1:]


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class _CudaView:
    """Expose library-owned device memory to torch via __cuda_array_interface__."""

    def __init__(self, ptr: int, shape, typestr: str, owner):
        self.__cuda_array_interface__ = {
            "shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}
        self._owner = owner


class _HostView:
    """Expose library-owned pinned host memory to numpy (and so to a CPU torch tensor) via __array_interface__."""

    def __init__(self, ptr: int, shape, typestr: str, owner):
        self.__array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 3}
        self._owner = owner


_TYPESTR = {torch.uint8: "|u1", torch.int32: "<i4", torch.int64: "<i8", torch.float32: "<f4",
            torch.float64: "<f8", torch.int8: "|i1", torch.int16: "<i2", torch.float16: "<f2"}


def alloc_rows(fields: Sequence[Field], n: int, device, names: Sequence[str] | None = None) -> dict:
    """n uninitialised rows of each named field (all when `names` is None), with the field's dtype and shape."""
    names = [f.name for f in fields] if names is None else list(names)
    return {f.name: torch.empty((n,) + tuple(f.shape), dtype=f.dtype, device=device)
            for f in fields if f.name in names}


class DeviceReplay:
    """`host_fields`: names of fields whose rows live in pinned, mapped host memory owned by the library
    (b2rl_replay_create_placed) instead of HBM: R2D2's `state`, which a step reads only for its sampled sequences.
    Their rows must be a multiple of 16 bytes.  gather() copies the sampled rows into device memory over PCIe,
    field_view() of such a field is a CPU tensor over the pinned rows, and conv1_fused / conv1_wgrad do not read them
    in place."""

    def __init__(self, capacity: int, fields: Sequence[Field] = APEX_FIELDS, device="cuda:0",
                 host_fields: Sequence[str] = ()):
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.B2RLError("DeviceReplay lives in GPU HBM; there is no CPU path")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.fields = tuple(fields)
        if len(self.fields) > _lib.MAX_FIELDS:
            raise ValueError("too many payload fields")
        self.capacity = int(capacity)
        d = ReplayDesc()
        d.capacity = self.capacity
        d.n_fields = len(self.fields)
        d.device = self.device.index
        for i, f in enumerate(self.fields):
            d.field_bytes[i] = f.nbytes
        names = [f.name for f in self.fields]
        unknown = set(host_fields) - set(names)
        if unknown:
            raise ValueError(f"host_fields names fields this replay does not have: {sorted(unknown)}")
        self.host_fields = frozenset(host_fields)
        on_host = (C.c_int32 * _lib.MAX_FIELDS)(*[int(n in self.host_fields) for n in names])
        torch.cuda.init()
        with torch.cuda.device(self.device):
            torch.zeros(1, device=self.device)  # make sure the primary context exists
        h = C.c_void_p()
        if self.host_fields:
            with hostmem.on_gpu_node(self.device):   # pinned pages on the GPU's NUMA node (first touch: the library)
                check(self.lib.b2rl_replay_create_placed(C.byref(d), on_host, C.byref(h)))
        else:
            check(self.lib.b2rl_replay_create(C.byref(d), C.byref(h)))
        self._h = h

    # -- bookkeeping -----------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self.lib.b2rl_replay_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _sizes(self):
        s, c, hd = C.c_int64(), C.c_int64(), C.c_int64()
        check(self.lib.b2rl_replay_size(self._h, C.byref(s), C.byref(c), C.byref(hd)))
        return s.value, c.value, hd.value

    def __len__(self) -> int:
        return self._sizes()[0]

    @property
    def head(self) -> int:
        return self._sizes()[2]

    def _st(self) -> int:
        return _stream_ptr(self.device)

    def field_view(self, name_or_idx) -> torch.Tensor:
        """Zero-copy torch view (capacity, *shape) of a library-owned payload field: a CUDA tensor, or for a host
        field a CPU tensor over its pinned rows (torch never treats host memory as device memory)."""
        i = name_or_idx if isinstance(name_or_idx, int) else [f.name for f in self.fields].index(name_or_idx)
        f = self.fields[i]
        p = C.c_void_p()
        check(self.lib.b2rl_replay_field_ptr(self._h, i, C.byref(p)))
        if f.name in self.host_fields:
            return torch.from_numpy(np.asarray(_HostView(p.value, (self.capacity,) + tuple(f.shape),
                                                         _TYPESTR[f.dtype], self)))
        view = _CudaView(p.value, (self.capacity,) + tuple(f.shape), _TYPESTR[f.dtype], self)
        with torch.cuda.device(self.device):
            return torch.as_tensor(view, device=self.device)

    # -- ingest ----------------------------------------------------------------
    def push(self, fields: Sequence, priorities) -> None:
        """fields[i]: tensor / ndarray (n, *shape_i), host (pinned preferred) or device."""
        keep = []
        ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
        n = None
        for i, (f, x) in enumerate(zip(self.fields, fields)):
            if x is None:
                ptrs[i] = None
                continue
            t = torch.as_tensor(x)
            if t.dtype != f.dtype:
                t = t.to(f.dtype)
            t = t.contiguous()
            if f.name in self.host_fields and not t.is_cuda and not t.is_pinned():
                # A host field is written in stream order (a host-to-host copy would not be): pageable rows are
                # staged in device memory on this stream, whose allocator reuses the staging in stream order.
                t = t.to(self.device)
            if n is None:
                n = t.shape[0]
            assert t.shape[0] == n and t.numel() * t.element_size() == n * f.nbytes, f"bad shape for {f.name}"
            keep.append(t)
            ptrs[i] = t.data_ptr()
        pr = torch.as_tensor(priorities).to(torch.float32).contiguous()
        if n is None:
            n = pr.shape[0]
        assert pr.numel() == n
        keep.append(pr)
        check(self.lib.b2rl_replay_push(self._h, ptrs, pr.data_ptr(), n, self._st()))
        # host buffers must outlive the async copies on this stream
        if any(not t.is_cuda and not t.is_pinned() for t in keep):
            pass  # pageable memory: cudaMemcpyAsync already staged it synchronously
        else:
            self._inflight = keep

    # -- pipelined ingest: H2D of the next batch overlaps the current learner step ------------
    def push_begin(self, fields: Sequence, n: int) -> None:
        """reserve (current stream) + payload copy on a private ingest stream.  Pair with push_commit."""
        if not hasattr(self, "_ingest_stream"):
            self._ingest_stream = torch.cuda.Stream(self.device)
            self._ev_reserved = torch.cuda.Event()
            self._ev_copied = torch.cuda.Event()
        start = C.c_int64()
        check(self.lib.b2rl_replay_reserve(self._h, int(n), C.byref(start), self._st()))
        self._ev_reserved.record(torch.cuda.current_stream(self.device))
        keep = []
        ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
        for i, (f, x) in enumerate(zip(self.fields, fields)):
            if x is None:
                ptrs[i] = None
                continue
            t = torch.as_tensor(x)
            assert t.dtype == f.dtype and t.is_contiguous() and t.numel() * t.element_size() == n * f.nbytes
            keep.append(t)
            ptrs[i] = t.data_ptr()
        with torch.cuda.stream(self._ingest_stream):
            self._ingest_stream.wait_event(self._ev_reserved)
            check(self.lib.b2rl_replay_copy_payload(self._h, ptrs, start.value, int(n),
                                                    self._ingest_stream.cuda_stream))
            self._ev_copied.record(self._ingest_stream)
        self._pending = (keep, int(n))

    def push_commit(self, priorities) -> None:
        """Make the records copied by push_begin sampleable (current stream waits for the copy)."""
        keep, n = self._pending
        pr = torch.as_tensor(priorities).to(torch.float32).contiguous()
        assert pr.numel() == n
        torch.cuda.current_stream(self.device).wait_event(self._ev_copied)
        check(self.lib.b2rl_replay_commit(self._h, pr.data_ptr(), n, self._st()))
        self._inflight = keep + [pr]
        self._pending = None

    def ingest_pipelined(self, fields: Sequence | None, priorities=None) -> None:
        """One C call per iteration (b2rl_replay_ingest_pipelined): publish the batch copied during the previous
        step, retire the next batch's slots, start its host->device copy on the library's copy stream.
        `fields`: pinned host (or device) tensors in field order, `priorities`: fp32[n]; fields None = flush."""
        if fields is None:
            check(self.lib.b2rl_replay_ingest_pipelined(self._h, None, None, 0, self._st()))
            self._pipe_keep = None
            return
        key = tuple(t.data_ptr() for t in fields) + (priorities.data_ptr(),)
        cache = getattr(self, "_pipe_cache", None)
        if cache is None or cache[0] != key:          # pointer array built once per set of staging buffers
            ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
            n = None
            for i, (f, t) in enumerate(zip(self.fields, fields)):
                assert t.dtype == f.dtype and t.is_contiguous()
                n = t.shape[0] if n is None else n
                assert t.numel() * t.element_size() == n * f.nbytes, f"bad shape for {f.name}"
                ptrs[i] = t.data_ptr()
            assert priorities.dtype == torch.float32 and priorities.numel() == n and priorities.is_contiguous()
            cache = self._pipe_cache = (key, ptrs, int(n))
        _, ptrs, n = cache
        check(self.lib.b2rl_replay_ingest_pipelined(self._h, ptrs, priorities.data_ptr(), n, self._st()))
        self._pipe_keep = (fields, priorities)        # host buffers stay alive until the next call

    def evict(self, delta: int) -> None:
        check(self.lib.b2rl_replay_evict(self._h, int(delta), self._st()))

    def fill_hash(self, n: int, seed: int = 0xB200) -> None:
        check(self.lib.b2rl_replay_fill_hash(self._h, int(n), int(seed) & 0xFFFFFFFF, self._st()))

    # -- tree ------------------------------------------------------------------
    def build(self, priorities: torch.Tensor) -> None:
        p = priorities.to(device=self.device, dtype=torch.float32).contiguous()
        check(self.lib.b2rl_tree_build(self._h, p.data_ptr(), p.numel(), self._st()))

    def seed(self, seed: int, counter: int = 0) -> None:
        """(Re)seed the device-resident Philox stream used when no uniforms are passed."""
        check(self.lib.b2rl_replay_seed(self._h, int(seed), int(counter), self._st()))

    def sample(self, n: int, beta: float = 0.4, u01: torch.Tensor | None = None,
               want_prob: bool = True, out=None, max_w: torch.Tensor | None = None):
        """-> (idx int64[n], prob fp32[n], weight fp32[n]) on the device.
        With explicit fp64 uniforms `u01` (parity runs) or, if None, from the
        handle's device-resident Philox stream (graph-replayable)."""
        if out is None:
            idx = torch.empty(n, dtype=torch.int64, device=self.device)
            prob = torch.empty(n, dtype=torch.float32, device=self.device) if want_prob else None
            w = torch.empty(n, dtype=torch.float32, device=self.device)
        else:
            idx, prob, w = out
        pp = prob.data_ptr() if prob is not None else None
        mw = max_w.data_ptr() if max_w is not None else None   # all-reduced max IS weight (multi-GPU)
        if u01 is not None:
            u01 = u01.to(device=self.device, dtype=torch.float64).contiguous()
            assert u01.numel() == n
            check(self.lib.b2rl_tree_sample(self._h, u01.data_ptr(), 0, 0, n, float(beta), mw,
                                            idx.data_ptr(), pp, w.data_ptr(), self._st()))
        else:
            check(self.lib.b2rl_tree_sample_stream(self._h, n, float(beta), mw, idx.data_ptr(), pp,
                                                   w.data_ptr(), self._st()))
        return idx, prob, w

    def sample_fetch(self, n: int, beta: float, idx: torch.Tensor, w: torch.Tensor, small: dict,
                     max_w: torch.Tensor | None = None, prob: torch.Tensor | None = None):
        """sample() from the device-resident Philox stream into the given buffers AND, in the same launch, copy
        the sampled slots' scalar fields (1/2/4/8-byte rows, e.g. action / reward / done) into `small[name]`.
        Everything is written in place, so a captured graph can prefetch the next minibatch's indices."""
        ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
        for i, f in enumerate(self.fields):
            t = small.get(f.name)
            ptrs[i] = t.data_ptr() if t is not None else None
        check(self.lib.b2rl_tree_sample_fetch(self._h, int(n), float(beta), max_w.data_ptr() if max_w is not None else None,
                                              idx.data_ptr(), prob.data_ptr() if prob is not None else None,
                                              w.data_ptr(), ptrs, self._st()))
        return idx, prob, w

    def sample_counter(self, seed: int, counter: int, n: int, beta: float = 0.4):
        """Stateless Philox draw: uniform k = philox(seed, counter + k)."""
        idx = torch.empty(n, dtype=torch.int64, device=self.device)
        prob = torch.empty(n, dtype=torch.float32, device=self.device)
        w = torch.empty(n, dtype=torch.float32, device=self.device)
        check(self.lib.b2rl_tree_sample(self._h, None, int(seed), int(counter), n, float(beta), None,
                                        idx.data_ptr(), prob.data_ptr(), w.data_ptr(), self._st()))
        return idx, prob, w

    def philox_uniforms(self, seed: int, offset: int, n: int) -> torch.Tensor:
        out = torch.empty(n, dtype=torch.float64, device=self.device)
        check(self.lib.b2rl_philox_uniforms(seed, offset, n, out.data_ptr(), self._st()))
        return out

    def update(self, idx: torch.Tensor, vals: torch.Tensor) -> None:
        idx = idx.to(device=self.device, dtype=torch.int64).contiguous()
        vals = vals.to(device=self.device, dtype=torch.float32).contiguous()
        assert idx.numel() == vals.numel()
        check(self.lib.b2rl_tree_update(self._h, idx.data_ptr(), vals.data_ptr(), idx.numel(), self._st()))

    def stats(self, beta: float = 0.4) -> torch.Tensor:
        """device tensor fp64[3] = {sum(p), min p, max IS weight}."""
        out = torch.empty(3, dtype=torch.float64, device=self.device)
        check(self.lib.b2rl_tree_stats(self._h, float(beta), out.data_ptr(), None, self._st()))
        return out

    def max_weight(self, beta: float = 0.4, out: torch.Tensor | None = None) -> torch.Tensor:
        """device fp32[1]: this shard's max IS weight (operand of the multi-GPU MAX all-reduce)."""
        out = torch.empty(1, dtype=torch.float32, device=self.device) if out is None else out
        check(self.lib.b2rl_tree_stats(self._h, float(beta), None, out.data_ptr(), self._st()))
        return out

    def priorities(self, start: int = 0, n: int | None = None) -> torch.Tensor:
        n = self.capacity - start if n is None else n
        out = torch.empty(n, dtype=torch.float32, device=self.device)
        check(self.lib.b2rl_tree_leaves(self._h, start, n, out.data_ptr(), self._st()))
        return out

    def tree_shape(self) -> tuple:
        """-> (cap2, G, top_bits): the tree's leaves (a power of two >= capacity), its stored internal levels and the
        binary levels its top group spans (b2rl_tree_level)."""
        n, g, tb = C.c_int64(), C.c_int32(), C.c_int32()
        check(self.lib.b2rl_tree_level(self._h, 0, C.byref(n), C.byref(g), C.byref(tb), None, None, None))
        return n.value, g.value, tb.value

    def tree_level(self, k: int) -> tuple:
        """Stored level k in 1..G of the sum-tree -> (sums fp64[n], mins fp32[n]) device tensors, n = cap2 >> 4k
        (1 at k = G: the root).  Level k holds the binary tree's nodes at height 4k; level 0, the leaves, is
        priorities()."""
        n = C.c_int64()
        check(self.lib.b2rl_tree_level(self._h, int(k), C.byref(n), None, None, None, None, None))
        sums = torch.empty(n.value, dtype=torch.float64, device=self.device)
        mins = torch.empty(n.value, dtype=torch.float32, device=self.device)
        check(self.lib.b2rl_tree_level(self._h, int(k), C.byref(n), None, None, sums.data_ptr(), mins.data_ptr(),
                                       self._st()))
        return sums, mins

    # -- gather ----------------------------------------------------------------
    def alloc_batch(self, n: int, names: Sequence[str] | None = None):
        return alloc_rows(self.fields, n, self.device, names)

    def gather(self, idx: torch.Tensor, out: dict | None = None) -> dict:
        n = idx.numel()
        if out is None:
            out = self.alloc_batch(n)
        ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
        for i, f in enumerate(self.fields):
            t = out.get(f.name)
            ptrs[i] = t.data_ptr() if t is not None else None
        check(self.lib.b2rl_replay_gather(self._h, idx.data_ptr(), n, ptrs, self._st()))
        return out

    def frame_source(self, name: str):
        """What conv1_fused / conv1_wgrad read frame field `name` from: its zero-copy view."""
        return self.field_view(name)

    def uniform_fetch(self, n: int, steps: int, out: dict) -> dict:
        """n distinct rollouts of `steps` steps drawn uniformly WITHOUT replacement from the valid region
        [head - size, head) (random.sample, baseline/utils.py:310-315) on the device-resident Philox stream, with
        the permutation of the served fill (b2rl_serve_fill_uniform), in ONE launch (b2rl_uniform_fetch) into the
        caller's fixed buffers: out["idx"] int64[n]; each non-frame field named in `out`, rows of `steps` words
        time-major (steps, n) and scalars (n,); out["rows"] (optional) int64[(steps + 1) * n], the rows of the
        time-major frames in the frame field viewed as one frame stack per row.  The frames are not copied.
        n > len(self) raises ValueError, as random.sample does, before anything is launched."""
        if n > len(self):
            raise ValueError("Sample larger than population")
        ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
        for i, f in enumerate(self.fields):
            t = out.get(f.name)
            if t is not None:
                assert t.is_contiguous() and t.numel() * t.element_size() == n * f.nbytes, f"bad buffer for {f.name}"
                ptrs[i] = t.data_ptr()
        idx, rows = out["idx"], out.get("rows")
        assert idx.dtype == torch.int64 and idx.is_contiguous() and idx.numel() == n
        assert rows is None or (rows.dtype == torch.int64 and rows.is_contiguous() and rows.numel() == (steps + 1) * n)
        check(self.lib.b2rl_uniform_fetch(self._h, int(n), int(steps), idx.data_ptr(), ptrs,
                                          None if rows is None else rows.data_ptr(), self._st()))
        return out


def dedup_pool_geometry(frames_per_slot: float, slots: int, window: int) -> tuple:
    """(pool frames F, window W) of a frame-deduplicated store: ceil(frames_per_slot * slots) frames, and `window`
    capped at an eighth of them, with a UserWarning when the cap applies.  A slot stays live until F - W frames have
    been stored after it, so the cap keeps that at least 7/8 of the pool (apex, r2d2 and impala.dedup_geometry)."""
    F = int(math.ceil(frames_per_slot * slots))
    W = min(int(window), F // 8)
    if W < window:
        warnings.warn(f"DEDUP_WINDOW = {window} frames is more than an eighth of the {F}-frame pool: the "
                      f"frame-deduplicated replay uses a window of {W} frames", stacklevel=3)
    return F, W


def coded_pool_bytes(frames_per_slot: float, slots: int, bytes_per_slot: float | None) -> int:
    """Bytes of a coded frame pool's ring: bytes_per_slot * slots rounded down to 16 bytes, or by default the raw size
    plus one frame, (F + 1) * 7 072 for dedup_pool_geometry's F, at which a slot dies by the byte rule no earlier than
    by the frame rule (DESIGN.md §4.21).  A smaller ring trades that for memory, at the mean stored bytes per frame
    codec_stats() reports (apex, r2d2 and impala.pool_bytes)."""
    if bytes_per_slot is None:
        return (int(math.ceil(frames_per_slot * slots)) + 1) * CODED_FRAME_BYTES
    return int(bytes_per_slot * slots) // 16 * 16


def check_codec_keys(cfg, codec: str, bytes_per_slot: str) -> None:
    """Refuse a learner config whose codec key `codec` is set without FRAME_DEDUP, or whose ring size key
    `bytes_per_slot` is set without `codec` or is not positive."""
    per = getattr(cfg, bytes_per_slot)
    if getattr(cfg, codec) and not cfg.FRAME_DEDUP:
        raise ValueError(f"{codec} encodes the frame pool of a FRAME_DEDUP store: set FRAME_DEDUP with it")
    if per is not None and not getattr(cfg, codec):
        raise ValueError(f"{bytes_per_slot} sizes the coded frame pool: set {codec} with it")
    if per is not None and not per > 0:
        raise ValueError(f"{bytes_per_slot} must be positive, not {per}")


class DedupReplay(DeviceReplay):
    """An Ape-X replay that stores every distinct frame once (b2rl_dedup_attach): slots hold APEX_DEDUP_FIELDS, the
    frames live in a pool of `pool_frames` frames, and a pushed frame reuses a stored one with the same content among
    the last `window` frames stored.  push / gather / sample / update / evict take and return what a DeviceReplay of
    APEX_FIELDS does, bit for bit; a slot also stops being live once pool_frames - window frames have been stored
    since its batch began (len() counts live slots).  The pipelined ingest forms are refused."""

    RECORD_FIELDS = APEX_FIELDS      # what push takes and gather returns
    coded = False                    # frames stored encoded (CodedDedupReplay, StripDedupReplay(pool_bytes=...))
    host_pool = False                # frames in pinned host memory (StripDedupReplay(host_pool=True))

    def __init__(self, capacity: int, pool_frames: int, window: int, device="cuda:0",
                 hash_mask: int = DEDUP_HASH_MASK):
        self._attach(capacity, APEX_DEDUP_FIELDS, device, "b2rl_dedup_attach", (), pool_frames, window, hash_mask)

    def _attach(self, capacity: int, fields, device, entry: str, lead: tuple, pool_frames: int, window: int,
                hash_mask: int, pool_bytes: int | None = None, host_pool: bool = False) -> None:
        """Every deduplicated store's constructor: the slot ring of `fields`, then the frame pool attached by the
        entry point `entry` (its _placed form with host_pool, its _coded form with pool_bytes) with the arguments
        `lead` between the planes field and pool_frames.  `pool` is the (F, 84, 84) frames on the device, a CPU
        tensor over them with host_pool, or the flat uint8 ring of 16-byte units of a coded pool, whose `offsets`
        are each entry's absolute unit offset."""
        DeviceReplay.__init__(self, capacity, fields, device)
        self.pool_frames, self.window = int(pool_frames), int(window)
        self.coded, self.host_pool = pool_bytes is not None, bool(host_pool)
        args = (self._h, 0, *lead, self.pool_frames, self.window, int(hash_mask))
        if self.host_pool:
            with hostmem.on_gpu_node(self.device):   # pinned pages on the GPU's NUMA node (first touch: the library)
                check(getattr(self.lib, entry + "_placed")(*args, 1))
        elif self.coded:
            check(getattr(self.lib, entry + "_coded")(*args, int(pool_bytes)))
        else:
            check(getattr(self.lib, entry)(*args))
        p, mb = C.c_void_p(), C.c_int64()
        check(self.lib.b2rl_dedup_info(self._h, C.byref(p), None, C.byref(mb)))
        self.max_batch = mb.value
        if self.host_pool:      # a CPU tensor over the pinned frames, as field_view of a host field
            on_host = C.c_int32()
            check(self.lib.b2rl_dedup_pool_placement(self._h, C.byref(on_host), C.byref(p)))
            self.pool = torch.from_numpy(np.asarray(_HostView(p.value, (self.pool_frames, 84, 84), "|u1", self)))
            return
        with torch.cuda.device(self.device):
            if not self.coded:
                self.pool = torch.as_tensor(_CudaView(p.value, (self.pool_frames, 84, 84), "|u1", self),
                                            device=self.device)
                return
            self.pool_bytes = int(pool_bytes)
            self.pool = torch.as_tensor(_CudaView(p.value, (self.pool_bytes,), "|u1", self), device=self.device)
            check(self.lib.b2rl_dedup_coded_offsets(self._h, C.byref(p)))
            self.offsets = torch.as_tensor(_CudaView(p.value, (self.pool_frames,), "<i8", self), device=self.device)

    def codec_stats(self) -> dict:
        """A coded pool's counters (b2rl_dedup_codec_stats): units_written (16-byte units, the wrap's skipped units
        included), pool_units, frames_stored, and bytes_per_frame = 16 units_written / frames_stored, the mean
        stored size of a frame (7 072 at most: raw)."""
        if not self.coded:
            raise ValueError("codec_stats() reports a coded frame pool (pool_bytes)")
        u, p, f = C.c_int64(), C.c_int64(), C.c_int64()
        check(self.lib.b2rl_dedup_codec_stats(self._h, C.byref(u), C.byref(p), C.byref(f)))
        return {"units_written": u.value, "pool_units": p.value, "frames_stored": f.value,
                "bytes_per_frame": 16.0 * u.value / f.value if f.value else 0.0}

    @property
    def head_seq(self) -> int:
        """Frames stored so far: the next new frame's sequence number (it goes to pool slot head_seq % pool_frames)."""
        h = C.c_int64()
        check(self.lib.b2rl_dedup_info(self._h, None, C.byref(h), None))
        return h.value

    def push(self, fields: Sequence, priorities) -> None:
        """fields: rows of RECORD_FIELDS, as for a DeviceReplay of them (host, pinned preferred, or device): Ape-X's
        [state, next_state, action, reward, done], R2D2's [state, ...] with `state` (n, T + 3, 84, 84) uint8 strips,
        IMPALA's [state, ...].  The frames are staged on the device (the same host->device bytes as a store without a
        frame pool), then pushed in chunks of at most max_batch records (b2rl_dedup_push, b2rl_dedup_push_strips);
        each chunk synchronizes the current stream once."""
        pr = torch.as_tensor(priorities).to(torch.float32).contiguous()
        n = pr.numel()
        framed = self._frame_fields
        small = _small_rows(self.RECORD_FIELDS[len(framed):], fields[len(framed):], n)
        frames = []
        for f, x in zip(framed, fields):
            t = torch.as_tensor(x)
            assert t.dtype == torch.uint8 and t.numel() == n * f.nbytes, \
                f"{f.name} must be uint8 ({n}, {', '.join(map(str, f.shape))})"
            frames.append(t.reshape(n, f.nbytes).to(self.device, non_blocking=True).contiguous())
        push = self.lib.b2rl_dedup_push if len(frames) == 2 else self.lib.b2rl_dedup_push_strips
        ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
        for a in range(0, n, self.max_batch):
            b = min(n, a + self.max_batch)
            ptrs[0] = None
            for i, t in enumerate(small):
                ptrs[1 + i] = t[a:b].data_ptr()
            check(push(self._h, *[t[a:b].data_ptr() for t in frames], ptrs, pr[a:b].data_ptr(), b - a, self._st()))
        self._inflight = frames + small + [pr]

    @property
    def _frame_fields(self) -> tuple:
        """The leading RECORD_FIELDS, whose frames live in the pool: the slot holds `planes` in their place."""
        return self.RECORD_FIELDS[:len(self.RECORD_FIELDS) + 1 - len(self.fields)]

    def push_begin(self, fields, n):
        raise ValueError("a frame-deduplicated replay (FRAME_DEDUP) has no pipelined ingest: use push")

    def ingest_pipelined(self, fields, priorities=None):
        raise ValueError("a frame-deduplicated replay (FRAME_DEDUP) has no pipelined ingest: use push")

    def fill_hash(self, n: int, seed: int = 0xB200):
        raise ValueError("a frame-deduplicated replay (FRAME_DEDUP) holds pool ids, not hashable payload")

    def alloc_batch(self, n: int, names: Sequence[str] | None = None):
        return alloc_rows(self.RECORD_FIELDS, n, self.device, names)

    def gather(self, idx: torch.Tensor, out: dict | None = None) -> dict:
        """The sampled slots' fields as a DeviceReplay of RECORD_FIELDS returns them, the frame fields assembled from
        the pool (b2rl_replay_gather_planes): Ape-X's (n, 4, 84, 84) state and next_state stacks, R2D2's (n, T + 3,
        84, 84) strips, IMPALA's (n, T + 1, 28 224) stacks; a coded pool's frames decoded."""
        n = idx.numel()
        if out is None:
            out = self.alloc_batch(n)
        frames = (C.c_void_p * 2)(*[_p(out.get(f.name)) for f in self._frame_fields])
        ptrs = (C.c_void_p * _lib.MAX_FIELDS)()
        for i, f in enumerate(self.fields):
            t = out.get(f.name) if i > 0 else None
            ptrs[i] = t.data_ptr() if t is not None else None
        check(self.lib.b2rl_replay_gather_planes(self._h, idx.data_ptr(), n, frames, ptrs, self._st()))
        return out

    def frame_source(self, name: str) -> "PlaneFrames":
        return PlaneFrames(self.pool, self.field_view("planes"), {"state": 0, "next_state": 4}[name])


def _small_rows(fields: Sequence[Field], xs: Sequence, n: int) -> list:
    """The non-frame fields of a dedup push as contiguous tensors of their fields' dtypes, n rows each."""
    out = []
    for f, x in zip(fields, xs):
        t = torch.as_tensor(x)
        t = (t if t.dtype == f.dtype else t.to(f.dtype)).contiguous()
        assert t.numel() * t.element_size() == n * f.nbytes, f"bad shape for {f.name}"
        out.append(t)
    return out


CODED_FRAME_BYTES = 7072      # the largest encoding of a frame: 16 header bytes and the 7 056 raw pixels


def _check_device_bytes(t, row: int, what: str) -> None:
    """The codec kernels read device uint8 rows of `row` bytes: refuse anything else before a launch."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8 or t.numel() % row != 0:
        desc = f"{t.dtype} {t.device} tensor of {t.numel()} elements" if isinstance(t, torch.Tensor) else type(t)
        raise ValueError(f"{what} must be a CUDA uint8 tensor of whole {row}-byte rows, not a {desc}")


def encode_frames(frames: torch.Tensor, stream=None) -> tuple:
    """The coded pool's encoding of each frame of a device uint8 (n, 84, 84) tensor (b2rl_frame_encode) -> (enc uint8
    (n, 7072), units int32 (n,)): frame j's encoding is enc[j, :16 units[j]]; the rest of the row is zero."""
    _check_device_bytes(frames, FRAME_BYTES, "frames")
    frames = frames.contiguous().view(-1, FRAME_BYTES)
    n = frames.shape[0]
    enc = torch.zeros(n, CODED_FRAME_BYTES, dtype=torch.uint8, device=frames.device)
    units = torch.empty(n, dtype=torch.int32, device=frames.device)
    st = torch.cuda.current_stream(frames.device).cuda_stream if stream is None else stream
    check(_lib.load().b2rl_frame_encode(frames.data_ptr(), n, enc.data_ptr(), units.data_ptr(), st))
    return enc, units


def decode_frames(enc: torch.Tensor, stream=None) -> torch.Tensor:
    """The inverse of encode_frames: a device uint8 (n, 7072) tensor of encodings -> (n, 84, 84) frames."""
    _check_device_bytes(enc, CODED_FRAME_BYTES, "encodings")
    enc = enc.contiguous().view(-1, CODED_FRAME_BYTES)
    out = torch.empty(enc.shape[0], 84, 84, dtype=torch.uint8, device=enc.device)
    st = torch.cuda.current_stream(enc.device).cuda_stream if stream is None else stream
    check(_lib.load().b2rl_frame_decode(enc.data_ptr(), enc.shape[0], out.data_ptr(), st))
    return out


class CodedDedupReplay(DedupReplay):
    """DedupReplay with its frames stored losslessly encoded (b2rl_dedup_attach_coded, ApexConfig.FRAME_CODEC, DESIGN.md
    §4.22): the pool is a device ring of pool_bytes holding each distinct frame's encoding (frame_codec.cuh), and a
    slot also dies once pool_bytes - 7072 (window + 1) bytes have been written since its batch began.  push / gather /
    sample / update take and return what a DedupReplay does, bit for bit, while every slot is live; gather() decodes
    the sampled s and s' stacks.  `pool` is the flat uint8 ring, and frame_source() is a CodedPlaneFrames: conv_1
    decodes each row's four frames on chip, so the sampled frames never pass through HBM decoded."""

    def __init__(self, capacity: int, pool_frames: int, window: int, pool_bytes: int, device="cuda:0",
                 hash_mask: int = DEDUP_HASH_MASK):
        self._attach(capacity, APEX_DEDUP_FIELDS, device, "b2rl_dedup_attach", (), pool_frames, window, hash_mask,
                     pool_bytes=pool_bytes)

    def frame_source(self, name: str) -> "CodedPlaneFrames":
        return CodedPlaneFrames(self.pool, self.field_view("planes"), self.offsets, self.pool_frames,
                                {"state": 0, "next_state": 4}[name])


class StripDedupReplay(DedupReplay):
    """The strip form of DedupReplay (b2rl_dedup_attach_strips, R2D2Config.FRAME_DEDUP, DESIGN.md §4.18): an R2D2
    replay whose slots hold R2D2_DEDUP_FIELDS(T), the T + 3 frames of each sequence's strip living in the frame pool.
    Sequences an actor cuts with half overlap (R2D2/Player.py:37-62) share about half of their frames, which are
    stored once.  push / gather / sample / update take and return what a DeviceReplay of r2d2_fields(T, strip=True)
    does, bit for bit, while every slot is live; the liveness rule and the refusals are DedupReplay's.
    `host_pool` (R2D2Config.HOST_POOL, DESIGN.md §4.19): the frame pool lives in pinned, mapped host memory owned by
    the library (b2rl_dedup_attach_strips_placed), allocated from a thread bound to the GPU's NUMA node; the planes,
    keys and sum-tree stay in HBM.  `pool` is then a CPU tensor, gather() copies the sampled strips over PCIe, and
    frame_source() is refused: conv_1 reads a gathered (staged) batch instead.
    `pool_bytes` (R2D2Config.POOL_CODEC, DESIGN.md §4.21): the frames are stored losslessly encoded in a device ring of
    pool_bytes (b2rl_dedup_attach_strips_coded), and a slot also dies once pool_bytes - 7072 (window + 1) bytes have
    been written since its batch began.  `pool` is then that flat uint8 ring, gather() decodes the sampled strips,
    codec_stats() reports the bytes stored per frame, and frame_source() is refused as for a host pool."""

    def __init__(self, capacity: int, pool_frames: int, window: int, T: int = 80, device="cuda:0",
                 hash_mask: int = DEDUP_HASH_MASK, hidden: int = 512, host_pool: bool = False,
                 pool_bytes: int | None = None):
        if host_pool and pool_bytes is not None:
            raise ValueError("a coded frame pool (pool_bytes) lives in HBM: it takes no host_pool")
        self.T = int(T)
        self.RECORD_FIELDS = r2d2_fields(self.T, hidden, strip=True)
        self._attach(capacity, R2D2_DEDUP_FIELDS(T, hidden), device, "b2rl_dedup_attach_strips", (self.T + 3,),
                     pool_frames, window, hash_mask, pool_bytes, host_pool)

    def frame_source(self, name: str) -> "PlaneFrames":
        """conv_1's rows of `state`: the windows of every slot's strip, row slot * (T + 3) + t being stack t of the
        slot (the row numbering of strip_windows over a strip store's state field)."""
        return _pool_rows(self, name, 1, "gather (decode) the sampled strips")


def _pool_rows(store, name: str, stride: int, read_first: str) -> "PlaneFrames":
    """conv_1's rows of a strip or rollout store's `state`: its plane table at `stride` over the pool.  Refused for a
    pool conv_1 cannot read in place, whose frames `read_first` brings into device memory instead."""
    if name != "state":
        raise KeyError(name)
    if store.coded:
        raise ValueError("conv_1 reads raw frame rows: a coded frame pool (pool_bytes) holds encoded frames and "
                         f"has no frame source; {read_first} into device memory first")
    if store.host_pool:
        raise ValueError("conv_1 reads its frame rows in place on the GPU: a frame pool in host memory (host_pool) "
                         "has no frame source; gather the sampled strips into device memory first")
    return PlaneFrames(store.pool, store.field_view("planes"), 0, stride)


class RolloutDedupReplay(StripDedupReplay):
    """The rollout form of StripDedupReplay (b2rl_dedup_attach_rollouts, ImpalaConfig.FRAME_DEDUP, DESIGN.md §4.20): an
    IMPALA replay whose slots hold IMPALA_DEDUP_FIELDS(T), the 4 (T + 1) frames of each rollout's T + 1 stacks living
    in the frame pool.  A stack repeats three frames of the one before it, a rollout's bootstrap stack is the first
    stack of the same actor's next rollout, and a rollout cut short at an episode end is padded with the previous
    rollout's stacks (IMPALA/Player.py:88-203), so about T of the 4 (T + 1) frames are new.  push / gather /
    uniform_fetch take and return what a DeviceReplay of impala_fields(T) does, bit for bit, while every slot is live;
    the liveness rule and the refusals are DedupReplay's, and the frame pool stays in HBM.
    `pool_bytes` (ImpalaConfig.STAGED_POOL_CODEC, DESIGN.md §4.23): the frames are stored losslessly encoded in a
    device ring of pool_bytes (b2rl_dedup_attach_rollouts_coded), and a slot also dies once pool_bytes - 7072 (window +
    1) bytes have been written since its batch began.  `pool` is then that flat uint8 ring, gather() and the served
    fill decode the sampled rollouts, codec_stats() reports the bytes stored per frame, frame_source() is refused, and
    stage_frames() decodes the distinct frames of drawn rollouts into a staged pool that conv_1 reads instead."""

    def __init__(self, capacity: int, pool_frames: int, window: int, T: int = 20, device="cuda:0",
                 hash_mask: int = DEDUP_HASH_MASK, pool_bytes: int | None = None):
        self.T = int(T)
        self.RECORD_FIELDS = impala_fields(self.T)
        self._attach(capacity, IMPALA_DEDUP_FIELDS(T), device, "b2rl_dedup_attach_rollouts", (self.T + 1,),
                     pool_frames, window, hash_mask, pool_bytes)

    def frame_source(self, name: str) -> "PlaneFrames":
        """conv_1's rows of `state`: every slot's stacks, row slot * (T + 1) + t being stack t of the slot (the row
        numbering of a stack store's state field viewed as (capacity * (T + 1), 4, 84, 84))."""
        return _pool_rows(self, name, 4, "stage the drawn rollouts (stage_frames)")

    def alloc_staged(self, n: int) -> dict:
        """stage_frames' buffers for n drawn rollouts, allocated once per learner: `pool` uint8 (n 4 (T + 1), 84, 84)
        and `planes` int32 (n, 4 (T + 1))."""
        R = 4 * (self.T + 1)
        return {"pool": torch.empty(n * R, 84, 84, dtype=torch.uint8, device=self.device),
                "planes": torch.empty(n, R, dtype=torch.int32, device=self.device)}

    def stage_frames(self, idx: torch.Tensor, staged: dict) -> "PlaneFrames":
        """The frames of the drawn slots idx (device int64 (n,), as uniform_fetch writes them) for conv_1, in one
        launch that a CUDA graph can capture (b2rl_dedup_stage_rollouts): each distinct frame of a rollout is decoded
        once into staged["pool"], and staged["planes"] names, for each of the rollout's 4 (T + 1) frames, the staged
        frame it equals.  -> the stride-4 PlaneFrames over them: row k (T + 1) + t is stack t of draw k, bit for bit
        what frame_source() of a raw store reads at row idx[k] (T + 1) + t."""
        if not self.coded:
            raise ValueError("stage_frames() decodes a coded frame pool (pool_bytes): read a raw pool through "
                             "frame_source()")
        n = idx.numel()
        pool, planes = staged["pool"], staged["planes"]
        if not (idx.is_cuda and idx.dtype == torch.int64 and idx.is_contiguous()):
            raise ValueError("idx must be a contiguous CUDA int64 tensor")
        R = 4 * (self.T + 1)
        if pool.dtype != torch.uint8 or not pool.is_contiguous() or pool.numel() != n * R * FRAME_BYTES or \
                planes.dtype != torch.int32 or not planes.is_contiguous() or planes.numel() != n * R:
            raise ValueError(f"staged buffers must be alloc_staged({n})'s: uint8 ({n * R}, 84, 84) and int32 "
                             f"({n}, {R})")
        check(self.lib.b2rl_dedup_stage_rollouts(self._h, idx.data_ptr(), n, pool.data_ptr(), planes.data_ptr(),
                                                 self._st()))
        return PlaneFrames(pool.view(n * R, 84, 84), planes.view(n, R), 0, 4)


# ---- stateless target kernels -------------------------------------------------
def _p(t):
    return None if t is None else t.data_ptr()


def apex_target(q_s, qn_online, qn_target, action, reward, notdone, weight, gamma_n, alpha,
                want_grad=True, out=None):
    """APE_X/Learner.py:85-121 in one launch.  All inputs device tensors."""
    lib = _lib.load()
    B, A = q_s.shape
    dev = q_s.device
    if out is None:
        out = {"target": torch.empty(B, device=dev), "td": torch.empty(B, device=dev),
               "prio": torch.empty(B, device=dev),
               "grad_q": torch.empty(B, A, device=dev) if want_grad else None,
               "scalars": torch.empty(3, device=dev)}
    action = action.to(torch.int64)
    for t in (q_s, qn_online, qn_target, action, reward, notdone, weight):
        assert t.is_cuda and t.is_contiguous()
    check(lib.b2rl_apex_target(_p(q_s), _p(qn_online), _p(qn_target), _p(action), _p(reward), _p(notdone),
                               _p(weight), B, A, float(np.float32(gamma_n)), float(alpha),
                               _p(out["target"]), _p(out["td"]), _p(out["prio"]), _p(out.get("grad_q")),
                               _p(out["scalars"]), _stream_ptr(dev)))
    return out


def r2d2_target(q, q_target, action, reward, notdone, weight, n_step, gamma, alpha, rescale=True,
                want_grad=True):
    """R2D2/Learner.py:110-198 in one launch (+ a 1-thread finisher for the scalars)."""
    lib = _lib.load()
    L, B, A = q.shape
    dev = q.device
    out = {"target": torch.empty(L - 1, B, device=dev), "td": torch.empty(L - 1, B, device=dev),
           "prio": torch.empty(B, device=dev),
           "grad_q": torch.empty(L, B, A, device=dev) if want_grad else None,
           "scalars": torch.empty(2, device=dev)}
    action = action.to(torch.int64).contiguous()
    check(lib.b2rl_r2d2_target(_p(q), _p(q_target), _p(action), _p(reward), _p(notdone), _p(weight),
                               L, B, A, int(n_step), float(gamma), float(alpha), int(bool(rescale)),
                               _p(out["target"]), _p(out["td"]), _p(out["prio"]), _p(out["grad_q"]),
                               _p(out["scalars"]), _stream_ptr(dev)))
    return out


def vtrace(pi_a, mu_a, value, bootstrap, reward, gamma, c_lambda, c_bar, p_bar):
    """IMPALA/Learner.py:141-215 in one launch.  (T, B) time-major."""
    lib = _lib.load()
    T, B = value.shape
    dev = value.device
    vt = torch.empty(T, B, device=dev)
    adv = torch.empty(T, B, device=dev)
    check(lib.b2rl_vtrace(_p(pi_a), _p(mu_a), _p(value), _p(bootstrap), _p(reward), T, B,
                          float(np.float32(gamma)), float(c_lambda), float(c_bar), float(p_bar),
                          _p(vt), _p(adv), _stream_ptr(dev)))
    return vt, adv


# ---- fused gather + first convolution (wgmma) -----------------------------------
class Conv1Pack:
    """Packed conv_1 weights of 1 or 2 networks for b2rl_conv1_fused (re-pack after every
    optimizer step of the online net / target sync: one tiny launch per network)."""

    def __init__(self, n_nets: int, device, c_out: int = 32):
        assert n_nets in (1, 2) and c_out in (16, 32)
        self.n_nets, self.c_out = n_nets, c_out
        self.device = torch.device(device)
        self.bq = torch.empty(n_nets * 4 * c_out * 256, dtype=torch.int8, device=self.device)
        self.scale = torch.empty(n_nets * c_out, dtype=torch.float32, device=self.device)

    def pack(self, net: int, weight: torch.Tensor) -> None:
        """weight: conv_1.weight fp32 (c_out, 4, 8, 8) (any memory format)."""
        w = weight.detach().to(torch.float32).contiguous(memory_format=torch.contiguous_format)
        assert w.shape == (self.c_out, 4, 8, 8)
        check(_lib.load().b2rl_conv1_pack(w.data_ptr(), net, self.n_nets, self.c_out, self.bq.data_ptr(),
                                          self.scale.data_ptr(), _stream_ptr(self.device)))


def conv1_pack_jobs(jobs) -> None:
    """jobs: up to 4 (pack, net, weight) triples -> ONE launch of all the packs (b2rl_conv1_pack_jobs)."""
    import ctypes as C
    n = len(jobs)
    ws = [w.detach().to(torch.float32).contiguous(memory_format=torch.contiguous_format) for _, _, w in jobs]
    c_out = jobs[0][0].c_out
    assert all(p.c_out == c_out and w.shape == (c_out, 4, 8, 8) for (p, _, _), w in zip(jobs, ws))
    arr = C.c_void_p * n
    check(_lib.load().b2rl_conv1_pack_jobs(
        arr(*[w.data_ptr() for w in ws]), (C.c_int32 * n)(*[net for _, net, _ in jobs]),
        (C.c_int32 * n)(*[p.n_nets for p, _, _ in jobs]), arr(*[p.bq.data_ptr() for p, _, _ in jobs]),
        arr(*[p.scale.data_ptr() for p, _, _ in jobs]), n, c_out, _stream_ptr(jobs[0][0].device)))


@dataclass(frozen=True)
class BoundFrames:
    """A frame source whose base address lives in device memory: entry `entry` of the int64 `table` holds the
    address of `rows` frame rows, `row_stride` bytes apart (b2rl_serve_bind writes it when a served minibatch slot is
    bound).  conv1_fused / conv1_wgrad read the entry when their kernels start, so a CUDA graph that captured them
    follows every rebind.  `row_stride`: FRAME_STACK_BYTES for frame stacks, FRAME_BYTES for the windows of frame
    strips (sequence_rows)."""
    table: torch.Tensor
    entry: int
    rows: int
    row_stride: int = FRAME_STACK_BYTES

    @property
    def device(self) -> torch.device:
        return self.table.device

    def entry_ptr(self) -> int:
        assert self.table.dtype == torch.int64 and self.table.is_contiguous() and 0 <= self.entry < self.table.numel()
        return self.table.data_ptr() + 8 * self.entry


@dataclass(frozen=True)
class PlaneFrames:
    """Frame stacks held as a plane table over a frame pool: row r is the stack whose channel c is pool frame
    planes.flatten()[plane_stride * r + base + c].  `pool`: uint8 (F, 84, 84).  DedupReplay: `planes` int32 (slots,
    8), plane_stride 8, `base` 0 for `state` and 4 for `next_state`.  StripDedupReplay: `planes` int32 (slots, T + 3),
    plane_stride 1, base 0, so row slot * (T + 3) + t is stack t of the slot's strip.  RolloutDedupReplay: `planes`
    int32 (slots, 4 (T + 1)), plane_stride 4, base 0, so row slot * (T + 1) + t is stack t of the slot's rollout.
    conv1_fused / conv1_wgrad read the four frames of each row in place."""
    pool: torch.Tensor
    planes: torch.Tensor
    base: int
    plane_stride: int = 8

    @property
    def device(self) -> torch.device:
        return self.pool.device

    @property
    def rows(self) -> int:
        """The rows whose four pool ids lie inside `planes`: every slot at stride 8, every stack at stride 4; at
        stride 1 every window but the last three, which would run past the table's end."""
        return (self.planes.numel() - self.base - 4) // self.plane_stride + 1


@dataclass(frozen=True)
class CodedPlaneFrames:
    """The Ape-X plane table over a coded frame pool (CodedDedupReplay.frame_source): row r is the stack whose channel
    c is the frame encoded at pool[16 (offsets[id % pool_frames] % (pool.numel() / 16)):], id = planes.flatten()[8 r +
    base + c].  `pool`: the flat uint8 ring; `offsets`: int64 (pool_frames,) descriptor table; `base` 0 for `state`,
    4 for `next_state`.  conv1_fused / conv1_wgrad decode each row's four frames in shared memory."""
    pool: torch.Tensor
    planes: torch.Tensor
    offsets: torch.Tensor
    pool_frames: int
    base: int

    @property
    def device(self) -> torch.device:
        return self.pool.device

    @property
    def rows(self) -> int:
        return (self.planes.numel() - self.base - 4) // 8 + 1


def _frame_source(frames) -> _lib.Frames:
    """The b2rl_frames descriptor of a frame tensor, a BoundFrames, a PlaneFrames or a CodedPlaneFrames.  A tensor's
    rows are its first dimension, each a contiguous FRAME_STACK_BYTES; stride(0) is the row stride (the library checks
    that it is a positive multiple of 16)."""
    if isinstance(frames, CodedPlaneFrames):
        if frames.pool.dim() != 1 or frames.pool.dtype != torch.uint8 or frames.pool.numel() % 16 != 0:
            raise ValueError("a coded frame pool is a flat uint8 ring of 16-byte units")
        if frames.pool.device.type != "cuda" or frames.offsets.device.type != "cuda":
            raise ValueError("conv_1 decodes a coded frame pool in place on the GPU: pool and offsets must be device "
                             "tensors")
        if frames.offsets.dtype != torch.int64 or frames.offsets.numel() != frames.pool_frames:
            raise ValueError("the descriptor table must be int64 (pool_frames,)")
        return _lib.Frames(pool=frames.pool.data_ptr(), planes=frames.planes.data_ptr(), plane_base=frames.base,
                           plane_stride=8, rows=frames.rows, offsets=frames.offsets.data_ptr(),
                           pool_units=frames.pool.numel() // 16, pool_frames=frames.pool_frames)
    if isinstance(frames, PlaneFrames):
        if frames.pool.dim() != 3:
            raise ValueError("conv_1 reads raw (F, 84, 84) pool frames: a coded frame pool holds encoded frames; "
                             "gather (decode) the sampled strips into device memory first")
        if frames.pool.device.type != "cuda":
            raise ValueError("conv_1 reads its frame rows in place on the GPU: a frame pool in host memory must be "
                             "gathered into device memory first")
        return _lib.Frames(pool=frames.pool.data_ptr(), planes=frames.planes.data_ptr(), plane_base=frames.base,
                           plane_stride=frames.plane_stride, rows=frames.rows)
    if isinstance(frames, BoundFrames):
        return _lib.Frames(table=frames.entry_ptr(), row_stride=frames.row_stride, rows=frames.rows)
    if frames.device.type != "cuda":
        raise ValueError("conv_1 reads its frame rows in place on the GPU: a frame source in host memory (a host "
                         "field's view) must be gathered into device memory first")
    assert frames.dtype == torch.uint8 and frames[0].is_contiguous() and frames[0].numel() == FRAME_STACK_BYTES
    stride = frames.stride(0) if frames.shape[0] > 1 else FRAME_STACK_BYTES   # a size-1 dimension's stride is arbitrary
    return _lib.Frames(base=frames.data_ptr(), row_stride=stride * frames.element_size(), rows=frames.shape[0])


def conv1_fused(frames, idx, pack: Conv1Pack, relu: bool = False, out=None):
    """frames: uint8 (rows, 4, 84, 84) with its inner three dimensions contiguous: frame stacks (e.g.
    DeviceReplay.field_view("state")), the windows of frame strips (strip_windows), a BoundFrames, a PlaneFrames
    (DedupReplay.frame_source, StripDedupReplay.frame_source, RolloutDedupReplay.frame_source) or a CodedPlaneFrames
    (CodedDedupReplay.frame_source);
    idx: int64[n] rows to take (None: all rows in order).
    -> list of n_nets tensors (n, c_out, 20, 20) fp32 in channels_last memory format."""
    src = _frame_source(frames)
    n = src.rows if idx is None else idx.numel()
    dev = frames.device
    if out is None:
        out = torch.empty((pack.n_nets, n, 20, 20, pack.c_out), dtype=torch.float32, device=dev)
    check(_lib.load().b2rl_conv1_fused(
        src, None if idx is None else idx.data_ptr(), n, pack.bq.data_ptr(), pack.scale.data_ptr(), pack.n_nets,
        pack.c_out, out.data_ptr(), int(bool(relu)), _stream_ptr(dev)))
    return [out[i].permute(0, 3, 1, 2) for i in range(pack.n_nets)]   # logical NCHW, physical NHWC


STEM_OUT, STEM_HW = 16, 42      # the stem's channels and pooled size (84 -> 42)


class StemPack:
    """Packed stem weights (the RESCNN2D node's first conv, 16 x 4 x 3 x 3) for b2rl_stem_fused: four signed 7-bit
    digits per weight and a per-channel scale, re-packed after every optimizer step (one tiny launch)."""

    BYTES = STEM_OUT * 4 * 48          # 3 072

    def __init__(self, device, bq: torch.Tensor | None = None, scale: torch.Tensor | None = None):
        """`bq`, `scale`: storage to pack into (stem_pack_pair's views), else freshly allocated."""
        self.device = torch.device(device)
        self.bq = torch.empty(self.BYTES, dtype=torch.int8, device=self.device) if bq is None else bq
        self.scale = torch.empty(STEM_OUT, dtype=torch.float32, device=self.device) if scale is None else scale

    def pack(self, weight: torch.Tensor) -> None:
        w = weight.detach().to(torch.float32).contiguous(memory_format=torch.contiguous_format)
        assert w.shape == (STEM_OUT, 4, 3, 3)
        check(_lib.load().b2rl_stem_pack(w.data_ptr(), self.bq.data_ptr(), self.scale.data_ptr(),
                                         _stream_ptr(self.device)))


def stem_fused(frames, idx, pack: StemPack, out=None):
    """The residual network's stem (3x3 conv of frames / 255, then a 3x3 / stride-2 max-pool) over rows `idx` of
    `frames` (any source conv1_fused takes, except a CodedPlaneFrames and an Ape-X plane table) -> (pooled fp32
    (n, 16, 42, 42), argmax uint8 (n, 16, 42, 42)): 3i + j of the first maximum of each window, row-major.
    `out`: a (pooled, argmax) pair to write into."""
    src = _frame_source(frames)
    n = src.rows if idx is None else idx.numel()
    dev = frames.device
    if out is None:
        out = (torch.empty((n, STEM_OUT, STEM_HW, STEM_HW), dtype=torch.float32, device=dev),
               torch.empty((n, STEM_OUT, STEM_HW, STEM_HW), dtype=torch.uint8, device=dev))
    pooled, amax = out
    assert pooled.is_contiguous() and amax.is_contiguous() and pooled.shape[0] == n and amax.shape[0] == n
    check(_lib.load().b2rl_stem_fused(src, None if idx is None else idx.data_ptr(), n, pack.bq.data_ptr(),
                                      pack.scale.data_ptr(), pooled.data_ptr(), amax.data_ptr(), _stream_ptr(dev)))
    return pooled, amax


def stem_pack_pair(device) -> tuple:
    """(online, target) StemPacks over one allocation, back to back as b2rl_stem_fused_pair reads them: a
    stem_fused_pair of the two then passes their storage as it lies."""
    bq = torch.empty(2 * StemPack.BYTES, dtype=torch.int8, device=device)
    scale = torch.empty(2 * STEM_OUT, dtype=torch.float32, device=device)
    return tuple(StemPack(device, bq[i * StemPack.BYTES:(i + 1) * StemPack.BYTES], scale[i * STEM_OUT:(i + 1) * STEM_OUT])
                 for i in range(2))


def stem_fused_pair(frames, idx, pack_online: StemPack, pack_target: StemPack, argmax: bool = True, out=None):
    """stem_fused of two networks over the same rows in one launch (b2rl_stem_fused_pair): each stack is read and
    zero-bordered once and run against both packs.  -> (online pooled, target pooled, online argmax or None), each
    net's pooled output (n, 16, 42, 42) and the argmax bit for bit stem_fused's with that pack.  `argmax`: write the
    online net's argmax (the grad pass needs it; the burn-in and the target never do).  Packs from stem_pack_pair are
    read in place; any other two are first copied side by side.  `out`: a (pooled (2, n, 16, 42, 42), argmax or None)
    pair to write into."""
    src = _frame_source(frames)
    n = src.rows if idx is None else idx.numel()
    dev = frames.device
    if out is None:
        out = (torch.empty((2, n, STEM_OUT, STEM_HW, STEM_HW), dtype=torch.float32, device=dev),
               torch.empty((n, STEM_OUT, STEM_HW, STEM_HW), dtype=torch.uint8, device=dev) if argmax else None)
    pooled, amax = out
    assert pooled.is_contiguous() and pooled.shape[:2] == (2, n) and (amax is None) == (not argmax)
    assert amax is None or (amax.is_contiguous() and amax.shape[0] == n)
    on, tg = pack_online, pack_target
    if tg.bq.data_ptr() == on.bq.data_ptr() + StemPack.BYTES and tg.scale.data_ptr() == on.scale.data_ptr() + 4 * STEM_OUT:
        bq, scale = on.bq, on.scale
    else:
        bq, scale = torch.cat([on.bq, tg.bq]), torch.cat([on.scale, tg.scale])
    check(_lib.load().b2rl_stem_fused_pair(src, None if idx is None else idx.data_ptr(), n, bq.data_ptr(),
                                           scale.data_ptr(), pooled.data_ptr(),
                                           None if amax is None else amax.data_ptr(), _stream_ptr(dev)))
    return pooled[0], pooled[1], amax


_stem_ws = {}


def stem_wgrad(frames, idx, gpooled: torch.Tensor, argmax: torch.Tensor, out: torch.Tensor | None = None,
               accumulate: bool = False) -> torch.Tensor:
    """dL/dW of the stem's conv from the same rows, dL/d(pooled) (n, 16, 42, 42) and stem_fused's argmax: the
    max-pool's backward folded into the kernel's loader (b2rl_stem_wgrad) -> (16, 4, 3, 3) fp32."""
    src = _frame_source(frames)
    n = src.rows if idx is None else idx.numel()
    shape = (n, STEM_OUT, STEM_HW, STEM_HW)
    assert gpooled.shape == shape and argmax.shape == shape and gpooled.dtype == torch.float32
    gpooled, argmax = gpooled.contiguous(), argmax.contiguous()
    dev = frames.device
    if dev not in _stem_ws:
        _stem_ws[dev] = torch.empty(_lib.load().b2rl_stem_wgrad_workspace_doubles(), dtype=torch.float64, device=dev)
    if out is None:
        out = torch.empty((STEM_OUT, 4, 3, 3), dtype=torch.float32, device=dev)
        accumulate = False
    assert out.is_contiguous() and out.numel() == STEM_OUT * 36
    check(_lib.load().b2rl_stem_wgrad(src, None if idx is None else idx.data_ptr(), n, gpooled.data_ptr(),
                                      argmax.data_ptr(), _stem_ws[dev].data_ptr(), out.data_ptr(),
                                      int(bool(accumulate)), _stream_ptr(dev)))
    return out


_wgrad_ws = {}


def conv1_wgrad(frames, idx, gy: torch.Tensor, out: torch.Tensor | None = None,
                accumulate: bool = False, relu_y: torch.Tensor | None = None) -> torch.Tensor:
    """dL/dW of conv_1 from the sampled uint8 rows and dL/dy, without staging the rows (b2rl_conv1_wgrad).
    frames: as for conv1_fused; idx: int64[n] or None; gy: (n, c_out, 20, 20) fp32
    (made channels_last if it is not) -> (c_out, 4, 8, 8) fp32.  relu_y: the post-ReLU output of
    conv1_fused(relu=True) for the same rows; gy is then dL/d(relu output) and is masked by (y > 0) in the kernel."""
    src = _frame_source(frames)
    n = src.rows if idx is None else idx.numel()
    c_out = gy.shape[1]
    assert gy.shape == (n, c_out, 20, 20) and gy.dtype == torch.float32
    gy = gy.contiguous(memory_format=torch.channels_last)
    if relu_y is not None:
        assert relu_y.shape == gy.shape and relu_y.dtype == torch.float32
        relu_y = relu_y.contiguous(memory_format=torch.channels_last)
    dev = frames.device
    key = (dev, c_out)
    if key not in _wgrad_ws:
        _wgrad_ws[key] = torch.empty(_lib.load().b2rl_conv1_wgrad_workspace_floats(c_out), dtype=torch.float32,
                                     device=dev)
    if out is None:
        out = torch.empty((c_out, 4, 8, 8), dtype=torch.float32, device=dev)
        accumulate = False
    assert out.is_contiguous() and out.numel() == c_out * 256
    check(_lib.load().b2rl_conv1_wgrad(
        src, None if idx is None else idx.data_ptr(), n, gy.data_ptr(), None if relu_y is None else relu_y.data_ptr(),
        c_out, _wgrad_ws[key].data_ptr(), out.data_ptr(), int(bool(accumulate)), _stream_ptr(dev)))
    return out
