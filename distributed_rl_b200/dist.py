"""Replay-sharded data parallelism helpers (SURVEY.md §8e).

The reference has a single learner process and no collective of any kind
(SURVEY §2 row 17); this is new work.  One process per GPU, slots sharded, every
rank samples locally; the ONLY inter-GPU traffic per step is
  * one all-reduce (mean) of the gradients, kept in one flat bucket, and
  * one all-reduce (max) of the shard's max IS weight ("priority-max reduction").
The helpers are backend-agnostic so the logic is covered by gloo tests on CPU.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def world() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


class FlatGradBucket:
    """All gradients of `params` as views into ONE contiguous buffer -> one collective per step."""

    def __init__(self, params, device=None, symmetric: bool = False):
        """symmetric=True: the bucket is a torch symmetric-memory allocation (every rank can map every other rank's
        bucket), which lets libb2rl's peer-memory all-reduce read the peers' gradients in place (csrc/peer.cu)."""
        self.params = list(params)
        device = device or self.params[0].device
        total = sum(p.numel() for p in self.params)
        padded = (total + 3) // 4 * 4
        self._symm = None
        if symmetric:
            try:
                import torch.distributed._symmetric_memory as symm
                self._flat_padded = symm.empty(padded, dtype=self.params[0].dtype, device=device)
                self._flat_padded.zero_()
                torch.cuda.synchronize(device)
                self._symm = symm.rendezvous(self._flat_padded, dist.group.WORLD)
            except Exception as e:                              # keep NCCL, loudly
                import warnings
                warnings.warn(f"symmetric gradient bucket unavailable ({e!r}); all-reduces stay on NCCL")
                self._symm = None
        if self._symm is None:
            self._flat_padded = torch.zeros(padded, device=device, dtype=self.params[0].dtype)
        self.flat = self._flat_padded[:total]
        off = 0
        for p in self.params:
            # same element order as the parameter (channels_last conv weights keep their strides), so that
            # elementwise fused optimizers can walk param and grad storage together
            p.grad = self.flat[off:off + p.numel()].as_strided(p.shape, p.stride())
            off += p.numel()

    def _reduce(self, t: torch.Tensor, async_op: bool = False):
        if dist.get_backend() == "nccl":
            return dist.all_reduce(t, op=dist.ReduceOp.AVG, async_op=async_op)
        w = dist.all_reduce(t, op=dist.ReduceOp.SUM, async_op=async_op)     # gloo has no AVG
        if not async_op:
            t.div_(world())
        return w

    def all_reduce_mean(self) -> None:
        if world() == 1:
            return
        self._reduce(self.flat)

    # -- overlap: reduce the gradients that are ready EARLY in the backward pass (the big head
    #    matrices, 97 % of the bytes) while the backward of the convolution stack still runs ----
    def enable_overlap(self, early_params, mid_params=()) -> None:
        """`early_params`: parameters whose gradients are complete first (the dense heads); `mid_params`: a second
        group that completes later but still well before the end of backward (conv_2 / conv_3: their weight
        gradients run on the sink's second lane) — each group is all-reduced as soon as its LAST gradient is
        reported, so only what is left (conv_1, 32 KB) is reduced after backward.  The bucket is re-laid
        early | mid | late; call finish() after backward."""
        def pick(sel):
            return [p for p in self.params if any(p is q for q in sel)]
        early, mid = pick(early_params), pick(mid_params)
        early.sort(key=lambda p: -p.numel())        # stable: equally shaped big matrices end up back to back, so one
        #                                             GEMM can write the sibling heads' gradients (linear._stacked_rows)
        late = [p for p in self.params if not any(p is q for q in early + mid)]
        self.params = early + mid + late
        off = 0
        for p in self.params:                       # re-lay the bucket: early params first
            p.grad = self.flat[off:off + p.numel()].as_strided(p.shape, p.stride())
            off += p.numel()
        n_early, n_mid = sum(p.numel() for p in early), sum(p.numel() for p in mid)
        self._early, self._late = self.flat[:n_early], self.flat[n_early + n_mid:]
        gloo = dist.is_initialized() and dist.get_backend() != "nccl"
        # one record per overlapped group: its slice, its parameters, the ids reported this step, the async work
        self._groups = [dict(flat=f, params=ps, ready=set(), work=None, div=False)
                        for f, ps in ((self._early, early), (self.flat[n_early:n_early + n_mid], mid)) if ps]
        self._group_of = {id(p): g for g in self._groups for p in g["params"]}
        self._sink_attached = False

        def mark(p):
            g = self._group_of.get(id(p))
            if g is None:
                return
            g["ready"].add(id(p))           # a set: a parameter reported twice still counts once
            if len(g["ready"]) == len(g["params"]) and g["work"] is None and world() > 1:
                big = getattr(self, "_peer_big", None)
                if big is not None and g is self._groups[0]:
                    big.mean_()                 # one libb2rl kernel on THIS stream (reduce-scatter + all-gather
                    g["work"] = True            # over NVLink peer memory): final for whatever follows on the stream
                else:
                    g["work"] = self._reduce(g["flat"], async_op=True)
                    g["div"] = gloo

        def autograd_hook(p):
            # torch >= 2.x runs post-accumulate-grad hooks even when a custom Function returned None for the
            # parameter (nothing was accumulated).  With a WeightGradSink attached the early gradients never come
            # through autograd — the sink reports them AFTER its own accumulation — so this path must stay silent,
            # or the all-reduce would start before the late-arriving gradients exist.
            if not self._sink_attached:
                mark(p)

        self._early_hook, self._early_params = mark, early + mid
        for p in early + mid:
            p.register_post_accumulate_grad_hook(autograd_hook)

    # the first group's handle under its old name (tests and diagnostics read it)
    @property
    def _work(self):
        gs = getattr(self, "_groups", [])
        return gs[0]["work"] if gs else None

    def enable_peer_allreduce(self) -> bool:
        """Reduce the late slice (what is left after backward: the critical-path collective) with libb2rl's
        peer-memory kernel instead of NCCL.  The slice is taken to the end of the bucket, which is padded to a
        multiple of 4 floats at construction.  Returns False (NCCL stays) where PeerAllReduce is not available."""
        if not hasattr(self, "_late") or not self._late.numel() or not PeerAllReduce.available(self.flat.device):
            return False
        if self._late.numel() > (1 << 20):                  # every rank reads world x slice: a small-message design
            return False
        start = self.flat.numel() - self._late.numel()
        start -= start % 4                                  # 16-byte aligned start: may take in the tail of a group
        self._late_padded = self._flat_padded[start:]       # ... whose own all-reduce completed before finish()
        import os
        import warnings
        try:
            self._peer = PeerAllReduce(self._late_padded.numel(), self.flat.device)
        except Exception as e:                              # no VMM / fabric support on this box: keep NCCL, loudly
            warnings.warn(f"peer-memory all-reduce unavailable ({e!r}); the late gradient slice stays on NCCL")
            self._peer = None
        # the early group (dense heads) in place in the symmetric bucket: reduce-scatter + all-gather kernel
        self._peer_big = None
        gs = getattr(self, "_groups", [])
        if self._peer is not None and self._symm is not None and gs and gs[0]["flat"].numel() % 4 == 0 \
                and gs[0]["flat"].data_ptr() == self._flat_padded.data_ptr() \
                and os.environ.get("B2RL_PEER_ALLREDUCE_BIG"):
            # opt-in: correct (tests/mgpu_worker.py), but at 2 ranks the kernel took 111 us against NCCL's 63 us
            # running beside backward at the lane's low priority (DESIGN.md §5)
            try:
                self._peer_big = PeerAllReduceBig(self._symm, gs[0]["flat"].numel(), self.flat.device)
            except Exception as e:
                warnings.warn(f"peer-memory all-reduce of the heads unavailable ({e!r}); they stay on NCCL")
        return self._peer is not None

    def attach_sink(self, sink) -> None:
        """Weight gradients that bypass autograd's AccumulateGrad (linear.WeightGradSink) report here instead:
        a group's all-reduce is then launched from the sink's side stream as soon as its last gradient
        has been accumulated there."""
        self._sink_attached = True
        for p in getattr(self, "_early_params", []):
            sink.on_ready[id(p)] = self._early_hook

    def wait_group(self, i: int = 0) -> bool:
        """Make the CURRENT stream wait for group i's all-reduce (launched by the hooks) and finish its mean.
        True if the group had been launched — its gradients are then final on this stream (the early optimizer
        step of the heads uses this); finish() will not wait for it again."""
        gs = getattr(self, "_groups", [])
        if i >= len(gs) or gs[i]["work"] is None:
            return False
        g = gs[i]
        if g["work"] is not True:
            g["work"].wait()
            if g["div"]:
                g["flat"].div_(world())
            g["work"] = True                # done: finish() will not wait again
        return True

    def finish(self) -> None:
        """After backward: reduce the late (small) part, then wait for the overlapped groups."""
        gs = getattr(self, "_groups", [])
        if world() == 1:
            for g in gs:
                g["ready"].clear()
            return
        if self._late.numel():
            if getattr(self, "_peer", None) is not None:
                self._peer.mean_(self._late_padded)          # one kernel over NVLink peer memory (csrc/peer.cu)
            else:
                self._reduce(self._late)
        for i, g in enumerate(gs):
            if g["work"] is None:                   # hooks did not fire (no such grads this step): reduce now
                self._reduce(g["flat"])
            else:
                self.wait_group(i)
            g["work"] = None
            g["ready"].clear()


class PeerAllReduce:
    """libb2rl's one-kernel mean all-reduce over NVLink peer memory (csrc/peer.cu) for ONE fixed slice size.
    Staging buffers and flag pads are torch symmetric-memory allocations (CUDA VMM handles exchanged through the
    process group's store), so every rank holds device pointers into every peer.  `available()` is False — and
    the caller keeps NCCL — off NCCL, across nodes, or when the rendezvous fails."""

    def __init__(self, n: int, device):
        import ctypes as C
        import torch.distributed._symmetric_memory as symm
        from . import _lib
        self._lib, self._C = _lib, C
        self.n = int(n)
        assert self.n % 4 == 0 and self.n >= 4
        self.device = torch.device(device)
        L = _lib.load()
        ctas = int(L.b2rl_peer_allreduce_max_ctas())
        w = world()
        group = dist.group.WORLD
        self.stage = symm.empty(2 * self.n, dtype=torch.float32, device=self.device)
        self.flags = symm.empty(w * ctas, dtype=torch.int32, device=self.device)
        self.flags.zero_()
        self.stage.zero_()
        torch.cuda.synchronize(self.device)
        hs, hf = symm.rendezvous(self.stage, group), symm.rendezvous(self.flags, group)
        self.rank, self.world = int(hs.rank), int(hs.world_size)
        self._stage_ptrs = torch.tensor(list(hs.buffer_ptrs), dtype=torch.int64, device=self.device)
        self._flag_ptrs = torch.tensor(list(hf.buffer_ptrs), dtype=torch.int64, device=self.device)
        self._epoch = torch.zeros(ctas, dtype=torch.int32, device=self.device)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._handles = (hs, hf)
        dist.barrier()                     # every pad is zeroed before any rank's first flag can land

    def mean_(self, t: torch.Tensor) -> torch.Tensor:
        """In place: t <- mean over ranks of t (t: contiguous fp32, numel == n, 16-byte aligned)."""
        assert t.numel() == self.n and t.is_contiguous() and t.dtype == torch.float32
        self._lib.check(self._lib.load().b2rl_peer_allreduce_mean(
            self._stage_ptrs.data_ptr(), self._flag_ptrs.data_ptr(), self.rank, self.world, self.n, t.data_ptr(),
            self.n, self._epoch.data_ptr(), self.error.data_ptr(),
            torch.cuda.current_stream(self.device).cuda_stream))
        return t

    @staticmethod
    def available(device) -> bool:
        import os
        if os.environ.get("B2RL_NO_PEER_ALLREDUCE") or not dist.is_initialized() or dist.get_backend() != "nccl":
            return False
        if world() < 2 or world() > 16 or torch.device(device).type != "cuda":
            return False
        # one node only: every rank must see every other rank's GPU as a peer
        local = int(os.environ.get("LOCAL_WORLD_SIZE", world()))
        return local == world() and torch.cuda.device_count() >= world()


class PeerAllReduceBig:
    """libb2rl's reduce-scatter + all-gather kernel (csrc/peer.cu k_peer_allreduce_big) over the first `n` floats of a
    symmetric gradient bucket (`handle`: its rendezvous).  mean_() leaves the rank-ordered mean in every rank's
    bucket, bit-identical across ranks, as ONE launch on the current stream."""

    CTAS = 32

    def __init__(self, handle, n: int, device):
        import torch.distributed._symmetric_memory as symm
        from . import _lib
        self._lib = _lib
        self.device = torch.device(device)
        self.n = int(n)
        self.rank, self.world = int(handle.rank), int(handle.world_size)
        self.slice = (self.n + 4 * self.world - 1) // (4 * self.world) * 4
        L = _lib.load()
        ctas = int(L.b2rl_peer_allreduce_max_ctas())
        self.result = symm.empty(2 * self.slice, dtype=torch.float32, device=self.device)
        self.flags = symm.empty(2 * self.world * ctas, dtype=torch.int32, device=self.device)
        self.result.zero_()
        self.flags.zero_()
        torch.cuda.synchronize(self.device)
        hr, hf = symm.rendezvous(self.result, dist.group.WORLD), symm.rendezvous(self.flags, dist.group.WORLD)
        mk = lambda ptrs: torch.tensor(list(ptrs), dtype=torch.int64, device=self.device)   # noqa: E731
        self._bucket_ptrs, self._result_ptrs, self._flag_ptrs = mk(handle.buffer_ptrs), mk(hr.buffer_ptrs), mk(hf.buffer_ptrs)
        self._epoch = torch.zeros(ctas, dtype=torch.int32, device=self.device)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._handles = (handle, hr, hf)
        dist.barrier()

    def mean_(self) -> None:
        self._lib.check(self._lib.load().b2rl_peer_allreduce_mean_big(
            self._bucket_ptrs.data_ptr(), self._result_ptrs.data_ptr(), self._flag_ptrs.data_ptr(), self.rank,
            self.world, self.n, self.slice, self.CTAS, self._epoch.data_ptr(), self.error.data_ptr(),
            torch.cuda.current_stream(self.device).cuda_stream))


def all_reduce_max_(x: torch.Tensor, async_op: bool = False):
    """In-place MAX all-reduce of the shard-local max IS weight.  async_op=True returns the work
    handle (None at world size 1) so the tiny collective can hide behind the learner step."""
    if world() > 1:
        w = dist.all_reduce(x, op=dist.ReduceOp.MAX, async_op=async_op)
        return w if async_op else x
    return None if async_op else x


def shard_slots(total_slots: int, rank: int, world_size: int) -> range:
    """Contiguous slot range owned by `rank` (SURVEY §8e 'contiguous ranges of N/G')."""
    per = (total_slots + world_size - 1) // world_size
    return range(min(rank * per, total_slots), min((rank + 1) * per, total_slots))
