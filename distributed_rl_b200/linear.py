"""Bias-free nn.Linear at fp32 accuracy on the tensor cores (3xTF32, csrc/gemm.cu).

The reference's dense heads are `nn.Linear(..., bias=False)` (baseline/baseNetwork.py:77-79); on the
GPU PyTorch runs them as fp32 SIMT GEMMs.  `linear3x(x, w)` computes the same `x @ w.T` — forward,
input gradient and weight gradient — with every operand split into two TF32 terms and three
wgmma products per term pair, fp32 accumulation in registers (error ~2^-22 relative per product,
the same order as an fp32 FMA chain; tests/test_gpu_03_gemm.py pins it against fp64).
"""
from __future__ import annotations

import contextlib

import torch

from . import _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


class SideBranch:
    """One fork/join site of a step on a side stream.  `with branch.fork():` runs its block on `stream` behind the
    work the current stream has queued so far (`after_current=False`: only behind what `stream` already holds);
    `join()` makes the current stream wait for every block forked since the last join.  With `stream=None`
    (parallelism disabled) the block runs in place and `join()` does nothing.  The events are created here, once,
    so that forking inside a captured step creates none."""

    def __init__(self, stream: torch.cuda.Stream | None):
        self.stream = stream
        self._forked, self._done = torch.cuda.Event(), torch.cuda.Event()
        self._open = False

    @contextlib.contextmanager
    def fork(self, after_current: bool = True):
        if self.stream is None:
            yield
            return
        if after_current:
            self._forked.record(torch.cuda.current_stream(self.stream.device))
            self.stream.wait_event(self._forked)
        with torch.cuda.stream(self.stream):
            yield
        self._done.record(self.stream)
        self._open = True

    def join(self) -> None:
        if self._open:
            torch.cuda.current_stream(self.stream.device).wait_event(self._done)
            self._open = False


class WeightGradSink:
    """Weight gradients off the critical path of backward.

    dL/dW of a layer feeds only the optimizer, while dL/dx feeds the rest of the backward pass.  Inside
    `with sink.active():` the layers of this module compute dL/dW on the sink's side stream, accumulate it into
    the (pre-allocated) `.grad` there and return None for it to autograd; `join()` makes the caller's stream
    wait for all of it (call it after backward, before the optimizer).  Tensors handed to the side stream are
    kept alive until the join, so their memory cannot be reused by the main stream while the side stream reads it.
    `on_ready` callbacks (e.g. the early gradient all-reduce of data parallelism) run on the side stream too."""

    def __init__(self, device):
        self.device = torch.device(device)
        # two lanes: the heads' weight gradients (the big GEMM + its operand packs) and the convolution stack's.
        # On one stream the conv_2 / conv_3 weight gradients queued behind the heads' and ran alone at the very end
        # of backward; on their own lane they overlap the dgrad chain.
        # Priorities (captured into the step's graph nodes): the learner's main branch runs at -2, the convolution
        # lane at -1 (its kernels must finish before the SM-filling conv_1 weight-gradient kernel starts), the
        # heads' lane (6.4 MB GEMM operands, the early optimizer step) at 0 fills what is left.
        self.lanes = (SideBranch(torch.cuda.Stream(self.device, priority=0)),
                      SideBranch(torch.cuda.Stream(self.device, priority=-1)))
        self._keep = []
        self._lane, self.accumulated = 0, (set(), set())   # per lane: ids of the params accumulated since the last join
        self.on_ready = {}          # id(param) -> callable, invoked (side stream) after that param's grad is complete

    @staticmethod
    def usable(params) -> bool:
        return _SINK is not None and all(p.grad is not None for p in params)

    def submit(self, fn, keep=(), lane: int = 0):
        self._lane = lane
        with self.lanes[lane].fork():
            fn()
        self._keep.extend(keep)

    def run_on_lane(self, fn, lane: int = 0):
        """Queue fn behind what the lane already holds, without a new dependency on the caller's stream."""
        with self.lanes[lane].fork(after_current=False):
            fn()

    def after_current(self, lane: int = 0):
        """The lane's later work waits for what the current stream has queued so far."""
        with self.lanes[lane].fork():
            pass

    def accumulate(self, param, grad):
        """(side stream) param.grad += grad, then the parameter's ready callback."""
        param.grad.add_(grad)
        self.written(param)

    def written(self, param):
        """(side stream) bookkeeping after param.grad received this backward's contribution."""
        self.accumulated[self._lane].add(id(param))
        cb = self.on_ready.get(id(param))
        if cb is not None:
            cb(param)

    # Set by a caller that guarantees every .grad is ZERO when backward starts (the fused optimizer zeroes them) and
    # that each parameter gets one contribution per backward: a layer may then WRITE its weight gradient into .grad
    # (e.g. as the output of its GEMM) instead of producing a temporary and adding it.
    grads_are_zero = False

    def join(self):
        for lane in self.lanes:
            lane.join()
        self._keep.clear()
        self.accumulated[0].clear()
        self.accumulated[1].clear()

    def active(self):
        return _SinkContext(self)


class _SinkContext:
    def __init__(self, sink):
        self.sink = sink

    def __enter__(self):
        global _SINK
        self._old, _SINK = _SINK, self.sink
        return self.sink

    def __exit__(self, *exc):
        global _SINK
        _SINK = self._old
        return False


_SINK: WeightGradSink | None = None


class OutputTape:
    """Record the outputs of the network's custom ops during one (no-grad) pass, or replay recorded outputs instead
    of recomputing them while a second pass only BUILDS the autograd graph.

    Use: the online network's two passes of an Ape-X step (Q(s) with grad, Q(s') without) run as ONE batched call
    under `OutputTape.record()`; the per-op outputs of the s half (`tape.half(n)`: views of the first n rows) are then
    replayed under `OutputTape.replay(...)` while `forward_from_conv1(y_s)` is called again with grad enabled: every
    op returns its recorded output (no kernel launch) and registers its normal backward.  The ops consult the tape in
    execution order: conv_2, act_2, conv_3, heads (ReLU + Flatten + first layers), dueling tail."""

    def __init__(self, mode, outs=None):
        self.mode, self.outs, self.pos = mode, ([] if outs is None else list(outs)), 0

    @staticmethod
    def record():
        return OutputTape("record")

    @staticmethod
    def replay(outs):
        return OutputTape("replay", outs)

    def half(self, n):
        return [t[:n] for t in self.outs]

    def __enter__(self):
        global _TAPE
        self._old, _TAPE = _TAPE, self
        return self

    def __exit__(self, *exc):
        global _TAPE
        _TAPE = self._old
        if self.mode == "replay" and exc[0] is None:
            assert self.pos == len(self.outs), "the replayed pass ran fewer ops than were recorded"
        return False


_TAPE: OutputTape | None = None


def taped(compute):
    """Output of one op: computed (and recorded) or taken from the tape."""
    t = _TAPE
    if t is None:
        return compute()
    if t.mode == "record":
        out = compute()
        t.outs.append(out)
        return out
    out = t.outs[t.pos]
    t.pos += 1
    return out


class _ReluTaped(torch.autograd.Function):
    """nn.ReLU whose output can come from the tape (backward: the usual mask on the output)."""

    @staticmethod
    def forward(ctx, x):
        y = taped(lambda: torch.relu(x))
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, gy):
        (y,) = ctx.saved_tensors
        return torch.ops.aten.threshold_backward(gy, y, 0)


def split_pack(x: torch.Tensor, transpose: bool, b_role: bool) -> torch.Tensor:
    """{hi, lo} TF32 operand image of a 2-D fp32 CUDA matrix (or of its transpose)."""
    if x.dim() != 2 or x.dtype != torch.float32 or not x.is_cuda:
        raise ValueError("split_pack expects a 2-D fp32 CUDA tensor")
    if x.stride(1) != 1:
        x = x.contiguous()
    rows, k = (x.shape[1], x.shape[0]) if transpose else (x.shape[0], x.shape[1])
    n = _lib.load().b2rl_gemm_packed_floats(rows, k, int(b_role))
    out = torch.empty(n, dtype=torch.float32, device=x.device)
    # a one-row matrix may carry any row stride (the transpose of an [n][1] column has stride 1): its rows are never
    # stepped, so give the pack the row length as the leading dimension
    ld = x.stride(0) if x.shape[0] > 1 else x.shape[1]
    _lib.check(_lib.load().b2rl_gemm_split_pack(x.data_ptr(), x.shape[0], x.shape[1], ld, int(transpose),
                                               int(b_role), out.data_ptr(), _stream()))
    return out


def pack_act_nhwc(y: torch.Tensor, transpose: bool) -> torch.Tensor:
    """Operand image of flatten_NCHW(relu(y)) (transpose=False: A-role, [B][C*HW]) or of its transpose
    (transpose=True: B-role) read straight from a channels_last (B, C, H, W) tensor — b2rl_gemm_pack_act_nhwc."""
    B, C, H, W = y.shape
    rows, k = (C * H * W, B) if transpose else (B, C * H * W)
    out = torch.empty(_lib.load().b2rl_gemm_packed_floats(rows, k, int(transpose)), dtype=torch.float32, device=y.device)
    _lib.check(_lib.load().b2rl_gemm_pack_act_nhwc(y.data_ptr(), B, H * W, C, 1, int(transpose), out.data_ptr(), _stream()))
    return out


def gemm_packed(a: torch.Tensor, b: torch.Tensor, M: int, N: int, K: int, out: torch.Tensor | None = None) -> torch.Tensor:
    """C[M][N] = A[M][K] @ B[N][K]^T from packed operand images (A-role, B-role)."""
    if out is None:
        n_pad = (N + 3) // 4 * 4
        out = torch.empty(M, n_pad, dtype=torch.float32, device=a.device)[:, :N]
    if out.stride(1) != 1 or out.stride(0) % 4:
        raise ValueError("output rows must be contiguous with a leading dimension divisible by 4")
    L = _lib.load()
    n_ws = L.b2rl_gemm_workspace_floats(M, N, K, out.stride(0))
    ws = torch.empty(n_ws, dtype=torch.float32, device=a.device) if n_ws else None
    _lib.check(L.b2rl_gemm_tf32x3(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, out.stride(0),
                                  ws.data_ptr() if ws is not None else None, _stream()))
    return out


def gemm_partials(a: torch.Tensor, b: torch.Tensor, M: int, N: int, K: int):
    """A[M][K] @ B[N][K]^T from packed operand images, left as its K-split partials (b2rl_gemm_tf32x3_partials):
    -> (partials, splits, ldc); partial z is rows [z*M, (z+1)*M) of partials viewed [splits*M][ldc].  Summed in
    split order they are gemm_packed's result, bit for bit."""
    L = _lib.load()
    ldc = (N + 3) // 4 * 4
    n_ws = L.b2rl_gemm_workspace_floats(M, N, K, ldc)
    splits = n_ws // (M * ldc) if n_ws else 1
    part = torch.empty(splits * M * ldc, dtype=torch.float32, device=a.device)
    _lib.check(L.b2rl_gemm_tf32x3_partials(a.data_ptr(), b.data_ptr(), part.data_ptr(), M, N, K, ldc, _stream()))
    return part, splits, ldc


def _pack_pieces(mats, transpose: bool, b_role: bool, out: torch.Tensor | None = None) -> torch.Tensor:
    """Operand image of vertically stacked matrices (transpose=False: rows stack) or of the transpose of
    that stack (transpose=True: the pieces sit side by side along the contraction index).  `out`: an existing
    image of that shape to overwrite."""
    L = _lib.load()
    inner, total = mats[0].shape[1], sum(m.shape[0] for m in mats)
    rows, k = (inner, total) if transpose else (total, inner)
    n = L.b2rl_gemm_packed_floats(rows, k, int(b_role))
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=mats[0].device)
    elif out.numel() != n or not out.is_contiguous():
        raise ValueError("`out` is not an image of this operand")
    off = 0
    for m in mats:
        if m.stride(1) != 1:
            m = m.contiguous()
        _lib.check(L.b2rl_gemm_split_pack_into(m.data_ptr(), m.shape[0], m.shape[1], m.stride(0), int(transpose),
                                               int(b_role), out.data_ptr(), rows, k,
                                               0 if transpose else off, off if transpose else 0, _stream()))
        off += m.shape[0]
    return out


class _Linear3x(torch.autograd.Function):
    """y = x @ cat(ws, 0).T for bias-free layers that share the input (one GEMM; the weights are never
    concatenated in memory: each is packed into its rows of the operand image).  `cache`: optional dict that
    keeps the packed forward operand between calls while the caller knows the weights are unchanged."""

    @staticmethod
    def forward(ctx, x, cache, *ws):
        M, K = x.shape
        N = sum(w.shape[0] for w in ws)
        b = cache.get("fwd") if cache is not None else None
        if b is None:
            b = _pack_pieces(ws, False, True)
            if cache is not None:
                cache["fwd"] = b
        y = gemm_packed(split_pack(x, False, False), b, M, N, K)
        ctx.save_for_backward(x, *ws)
        ctx.cache = cache
        return y

    @staticmethod
    def backward(ctx, gy):
        x, *ws = ctx.saved_tensors
        M, K = x.shape
        N = sum(w.shape[0] for w in ws)
        gy = gy.contiguous()
        gx, gws = None, [None] * len(ws)
        if any(ctx.needs_input_grad[2:]):
            # dW[N][K] = gy^T[N][M] @ x[M][K]: contraction over M.  Submitted before dx is launched, so the sink's
            # lane forks from the stream as it is now and runs beside the dx GEMM, not behind it.
            def wgrad():
                gw = gemm_packed(split_pack(gy, True, False), split_pack(x, True, True), N, K, M)
                return list(torch.split(gw, [w.shape[0] for w in ws], 0))
            if WeightGradSink.usable(ws):
                sink = _SINK

                def deferred():
                    for w, g in zip(ws, wgrad()):
                        sink.accumulate(w, g)
                sink.submit(deferred, keep=(gy, x))
            else:
                gws = wgrad()
        if ctx.needs_input_grad[0]:
            # dx[M][K] = gy[M][N] @ W[N][K]: contraction over N, the B operand is W^T ([K rows][N])
            bt = ctx.cache.get("bwdT") if ctx.cache is not None else None     # prepared ahead (GraphAgent.prepack_heads)
            gx = gemm_packed(split_pack(gy, False, False), bt if bt is not None else _pack_pieces(ws, True, True), M, K, N)
            _images_read()
        return (gx, None, *gws)


class _ReluFlatLinear3x(torch.autograd.Function):
    """h = flatten_NCHW(relu(y)) @ cat(ws, 0).T for a conv output `y` (B, C, H, W) stored channels_last, WITHOUT the
    ReLU kernel, the NHWC -> NCHW flatten copy and their backward counterparts: the activation-side packs read y
    coalesced, apply the ReLU, transpose through shared memory and write the operand images in the weights'
    NCHW-flatten feature order (csrc/gemm.cu k_pack_act_nhwc); dL/dy comes back through one unflatten + ReLU-mask
    kernel.  The weights' packs are the ordinary ones (shared with _Linear3x: cache keys "fwd" / "bwdT").
    Same arithmetic as act_3 + nn.Flatten + _Linear3x (cfg/ape_x.json:37-71), operand for operand."""

    @staticmethod
    def forward(ctx, y, cache, *ws):
        B, C, H, W = y.shape
        N, K = sum(w.shape[0] for w in ws), C * H * W
        b = cache.get("fwd") if cache is not None else None
        if b is None:
            b = _pack_pieces(ws, False, True)
            if cache is not None:
                cache["fwd"] = b
        h = taped(lambda: gemm_packed(pack_act_nhwc(y, False), b, B, N, K))
        ctx.save_for_backward(y, *ws)
        ctx.cache = cache
        return h

    @staticmethod
    def backward(ctx, gh):
        y, *ws = ctx.saved_tensors
        gy, gws = _relu_flat_backward(y, ws, ctx.cache, gh, ctx.needs_input_grad[0], any(ctx.needs_input_grad[2:]))
        return (gy, None, *gws)


def _relu_flat_backward(y, ws, cache, gh, need_gy: bool, need_gw: bool):
    """Backward of h = flatten_NCHW(relu(y)) @ cat(ws, 0).T -> (dL/dy or None, [dL/dW_i or None]).  The weight
    gradients go to the active WeightGradSink when there is one."""
    B, C, H, W = y.shape
    N, K = sum(w.shape[0] for w in ws), C * H * W
    gh = gh.contiguous()
    gy, gws = None, [None] * len(ws)
    if need_gw:
        def wgrad():
            gw = gemm_packed(split_pack(gh, True, False), pack_act_nhwc(y, True), N, K, B)
            return list(torch.split(gw, [w.shape[0] for w in ws], 0))
        if WeightGradSink.usable(ws):       # before dL/dy is launched: runs beside it (see _Linear3x.backward)
            sink = _SINK

            def deferred():
                joint = _stacked_rows([w.grad for w in ws]) if sink.grads_are_zero else None
                if joint is not None and not any(id(w) in sink.accumulated[0] for w in ws):
                    # the GEMM writes dW of all sibling heads straight into their (adjacent, zero) .grad rows:
                    # no temporary and no 6.4 MB grad.add_ per head (the heads' all-reduce starts that much earlier)
                    gemm_packed(split_pack(gh, True, False), pack_act_nhwc(y, True), N, K, B, out=joint)
                    for w in ws:
                        sink.written(w)
                else:
                    for w, g in zip(ws, wgrad()):
                        sink.accumulate(w, g)
            sink.submit(deferred, keep=(gh, y))
        else:
            gws = wgrad()
    if need_gy:
        bt = cache.get("bwdT") if cache is not None else None
        # dL/dx stays as its K-split partials: the unflatten + ReLU-mask kernel sums them while it reads them
        gx, splits, ld = gemm_partials(split_pack(gh, False, False), bt if bt is not None else _pack_pieces(ws, True, True),
                                       B, K, N)
        gy = torch.empty_like(y)                                         # channels_last like y
        _lib.check(_lib.load().b2rl_unflatten_relu_mask(gx.data_ptr(), ld, splits, B * ld, y.data_ptr(), B, H * W, C,
                                                       gy.data_ptr(), _stream()))
        _images_read()
    return gy, gws


def _images_read():
    """dL/dx of the heads has been issued.  The heads' lane steps their weights early (FusedRMSprop.step_early), and
    that update rewrites the weights' resident W^T operand image the dL/dx GEMM reads: order the lane behind it."""
    if _SINK is not None:
        _SINK.after_current(0)


def _stacked_rows(ts):
    """One (sum rows, K) view over 2-D fp32 tensors that lie back to back in one storage (the flat gradient buffer
    lays the heads' first-layer gradients out that way), else None."""
    t0 = ts[0]
    if not all(t is not None and t.dim() == 2 and t.is_contiguous() and t.dtype == torch.float32
               and t.shape[1] == t0.shape[1] for t in ts):
        return None
    off = t0.data_ptr()
    for t in ts:
        if t.data_ptr() != off:
            return None
        off += t.numel() * 4
    end = t0.storage_offset() + sum(t.numel() for t in ts)
    if end * 4 > t0.untyped_storage().nbytes() or t0.shape[1] % 4:
        return None
    return t0.as_strided((sum(t.shape[0] for t in ts), t0.shape[1]), (t0.shape[1], 1))


def relu_flat_linear3x(y: torch.Tensor, ws, cache: dict | None = None) -> torch.Tensor:
    """See _ReluFlatLinear3x.  `y`: (B, C, H, W) fp32 CUDA, channels_last-contiguous, PRE-ReLU conv output."""
    return _ReluFlatLinear3x.apply(y, cache, *ws)


def relu_flat_supported(y: torch.Tensor, ws) -> bool:
    return (y.is_cuda and y.dim() == 4 and y.dtype == torch.float32
            and y.is_contiguous(memory_format=torch.channels_last)
            and y.shape[2] * y.shape[3] * (y.shape[1] + 1) * 4 <= 48 * 1024
            and all(w.dim() == 2 and w.shape[1] == y.shape[1] * y.shape[2] * y.shape[3] for w in ws)
            and not any(w.shape[0] % 32 for w in ws[:-1]))


def linear3x(x: torch.Tensor, w, cache: dict | None = None) -> torch.Tensor:
    """`torch.nn.functional.linear(x, w)` for 2-D fp32 CUDA `x` ([M][K]) and bias-free `w` ([N][K]); `w` may be
    a list of weights sharing the input (their outputs are concatenated along the last dimension).  Inner
    pieces of a list must have a multiple of 32 rows."""
    ws = [w] if torch.is_tensor(w) else list(w)
    if len(ws) > 1 and any(m.shape[0] % 32 for m in ws[:-1]):
        ws = [torch.cat(ws, 0)]
    return _Linear3x.apply(x, cache, *ws)


class _DuelingTail(torch.autograd.Function):
    """Q = relu(h[:, :H]) @ Wa.T + relu(h[:, H:]) @ Wv.T - mean_j(adv_j)  in one kernel (csrc/dueling.cu)."""

    @staticmethod
    def forward(ctx, h, wa, wv):
        M, H2 = h.shape
        A, H = wa.shape

        def compute():
            q = torch.empty(M, A, dtype=torch.float32, device=h.device)
            _lib.check(_lib.load().b2rl_dueling_forward(h.data_ptr(), 1, 0, M, H, wa.data_ptr(), A, wv.data_ptr(),
                                                        q.data_ptr(), None, _stream()))
            return q
        q = taped(compute)
        ctx.save_for_backward(h, wa, wv)
        return q

    @staticmethod
    def backward(ctx, gq):
        h, wa, wv = ctx.saved_tensors
        return _dueling_backward(h, wa, wv, gq, ctx.needs_input_grad[0], ctx.needs_input_grad[1] or ctx.needs_input_grad[2])


def _dueling_backward(h, wa, wv, gq, need_gh: bool, need_w: bool):
    """Backward of the dueling tail -> (dL/dh, dL/dWa, dL/dWv); each None when not needed, the weights' also when
    the active WeightGradSink takes them."""
    M, H2 = h.shape
    A, H = wa.shape
    gq = gq.contiguous()
    gh = torch.empty_like(h) if need_gh else None
    L = _lib.load()
    row_ws = torch.empty(M * (A + 1), dtype=torch.float32, device=h.device)
    defer = need_w and WeightGradSink.usable((wa, wv))
    gwa = torch.empty_like(wa) if need_w else None
    gwv = torch.empty_like(wv) if need_w else None
    # row pass (dL/dh + the per-row table) on this stream; the column pass (dL/dW) here or on the sink's stream
    _lib.check(L.b2rl_dueling_backward(h.data_ptr(), gq.data_ptr(), M, H, wa.data_ptr(), A, wv.data_ptr(),
                                       gh.data_ptr() if gh is not None else None,
                                       None if (defer or not need_w) else gwa.data_ptr(),
                                       None if (defer or not need_w) else gwv.data_ptr(), row_ws.data_ptr(), _stream()))
    if defer:
        sink = _SINK

        def deferred():
            _lib.check(L.b2rl_dueling_backward_w(h.data_ptr(), row_ws.data_ptr(), M, H, A, gwa.data_ptr(),
                                                 gwv.data_ptr(), _stream()))
            sink.accumulate(wa, gwa)
            sink.accumulate(wv, gwv)
        sink.submit(deferred, keep=(h, row_ws, gwa, gwv))
        return gh, None, None
    return gh, gwa, gwv


class _ReluFlatHeadsDueling(torch.autograd.Function):
    """Q = dueling_tail(relu_flat_linear3x(y, ws), wa, wv) with the heads' GEMM left as its K-split partials, which
    the dueling forward kernel sums while it stages its rows (no k_splitk_reduce launch, no h round trip through it).
    h is written only when backward or the tape needs it.  Tape: h, then q, like the two ops it replaces.  Backward:
    the two ops' backward bodies, in their order."""

    @staticmethod
    def forward(ctx, y, cache, need_h, wa, wv, *ws):
        B, C, Hh, W = y.shape
        N, K = sum(w.shape[0] for w in ws), C * Hh * W
        A, H = wa.shape
        b = cache.get("fwd") if cache is not None else None
        if b is None:
            b = _pack_pieces(ws, False, True)
            if cache is not None:
                cache["fwd"] = b
        res = {}

        def heads():
            part, splits, ldc = gemm_partials(pack_act_nhwc(y, False), b, B, N, K)
            h = torch.empty(B, N, dtype=torch.float32, device=y.device) if need_h else None
            q = torch.empty(B, A, dtype=torch.float32, device=y.device)
            _lib.check(_lib.load().b2rl_dueling_forward(part.data_ptr(), splits, B * ldc, B, H, wa.data_ptr(), A,
                                                        wv.data_ptr(), q.data_ptr(),
                                                        h.data_ptr() if h is not None else None, _stream()))
            res["q"] = q
            return h
        h = taped(heads)
        q = taped(lambda: res["q"])
        ctx.save_for_backward(y, h, wa, wv, *ws)
        ctx.cache = cache
        return q

    @staticmethod
    def backward(ctx, gq):
        y, h, wa, wv, *ws = ctx.saved_tensors
        need = ctx.needs_input_grad
        need_gy, need_gws = need[0], any(need[5:])
        gh, gwa, gwv = _dueling_backward(h, wa, wv, gq, need_gy or need_gws, need[3] or need[4])
        gy, gws = (_relu_flat_backward(y, ws, ctx.cache, gh, need_gy, need_gws) if gh is not None
                   else (None, [None] * len(ws)))
        return (gy, None, None, gwa, gwv, *gws)


def relu_flat_heads_dueling(y: torch.Tensor, ws, wa: torch.Tensor, wv: torch.Tensor, cache: dict | None = None):
    """dueling_tail(relu_flat_linear3x(y, ws, cache), wa, wv) as one op (see _ReluFlatHeadsDueling)."""
    need_h = torch.is_grad_enabled() or _TAPE is not None
    return _ReluFlatHeadsDueling.apply(y, cache, need_h, wa, wv, *ws)


def dueling_tail_supported(h: torch.Tensor, wa: torch.Tensor, wv: torch.Tensor) -> bool:
    return (h.is_cuda and h.dim() == 2 and h.dtype == torch.float32 and h.is_contiguous()
            and wa.dim() == 2 and wv.shape == (1, wa.shape[1]) and h.shape[1] == 2 * wa.shape[1]
            and wa.shape[1] % 32 == 0 and wa.shape[1] <= 1024 and wa.shape[0] <= 32
            and wa.is_contiguous() and wv.is_contiguous())


def dueling_tail(h: torch.Tensor, wa: torch.Tensor, wv: torch.Tensor) -> torch.Tensor:
    """h: [M][2H] pre-activations of the two heads' first layers (advantage | value); wa: [A][H]; wv: [1][H]."""
    return _DuelingTail.apply(h, wa, wv)
