"""FusedRMSprop — torch.optim.RMSprop's update for the learners' configs (cfg/ape_x.json centered,
cfg/impala.json plain) as one libb2rl launch that also zeroes the gradients and produces the
reference's diagnostic gradient "norm" (APE_X/Learner.py:123-138).  momentum and weight_decay are
0 in every shipped config and are not supported here (falls back to torch.optim.RMSprop)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import check


class FusedRMSprop:
    def __init__(self, params, lr, alpha=0.99, eps=1e-8, centered=False):
        self.params = [p for p in params]
        assert 1 <= len(self.params) <= 24
        self.lr, self.alpha, self.eps, self.centered = float(lr), float(alpha), float(eps), bool(centered)
        dev = self.params[0].device
        self.device = dev
        for p in self.params:
            assert p.is_cuda and p.dtype == torch.float32 and _dense(p), "dense fp32 CUDA parameters only"
            if p.grad is None or p.grad.stride() != p.stride():
                # gradients must share the parameter's element order (channels_last weights!): autograd
                # accumulates in place into this buffer from then on
                old = p.grad
                p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
                if old is not None:
                    p.grad.copy_(old)
        self.square_avg = [torch.zeros_like(p, memory_format=torch.preserve_format) for p in self.params]
        self.grad_avg = [torch.zeros_like(p, memory_format=torch.preserve_format) for p in self.params] \
            if self.centered else None
        n = len(self.params)
        self._scratch = torch.zeros(n, dtype=torch.float64, device=dev)
        self.grad_norm = torch.zeros(1, dtype=torch.float32, device=dev)
        arr = C.c_void_p * n
        self._p = arr(*[p.data_ptr() for p in self.params])
        self._sq = arr(*[t.data_ptr() for t in self.square_avg])
        self._ga = arr(*[t.data_ptr() for t in self.grad_avg]) if self.centered else None
        self._numel = (C.c_int64 * n)(*[p.numel() for p in self.params])
        self._arr = arr
        self._images = [(0,) * 6 for _ in self.params]     # see write_images
        self._keep_images = []

    def write_images(self, param, fwd: torch.Tensor, wt: torch.Tensor | None, total_n: int, n_off: int) -> None:
        """From now on every update of `param` (rows x cols, row-major) also writes it into the 3xTF32 B-role operand
        images of the weight stack it belongs to (total_n rows, `param` at row n_off): `fwd` of the stack, `wt` (may
        be None) of its transpose — the images linear._pack_pieces(stack, False / True, True) builds.  The images
        must be current when this is called; the update keeps them so."""
        i = next(i for i, p in enumerate(self.params) if p is param)
        rows, cols = param.shape
        assert param.is_contiguous() and param.grad.is_contiguous()
        self._images[i] = (fwd.data_ptr(), wt.data_ptr() if wt is not None else 0, rows, cols, total_n, n_off)
        self._keep_images.extend([fwd, wt])

    def _launch(self, lo: int, hi: int, norm_out) -> None:
        """Update + zero_grad of tensors [lo, hi); their squared gradient norms land in scratch slots [lo, hi)."""
        n = hi - lo
        sub = lambda a: (C.c_void_p * n)(*a[lo:hi])       # noqa: E731
        for p in self.params[lo:hi]:
            assert p.grad.stride() == p.stride()
        check(_lib.load().b2rl_rmsprop_step(
            sub(self._p), (C.c_void_p * n)(*[p.grad.data_ptr() for p in self.params[lo:hi]]), sub(self._sq),
            sub(self._ga) if self.centered else None, (C.c_int64 * n)(*self._numel[lo:hi]), n, self.lr, self.alpha,
            self.eps, int(self.centered), (C.c_int64 * (6 * n))(*[v for im in self._images[lo:hi] for v in im]),
            self._scratch.data_ptr() + 8 * lo, norm_out,
            torch.cuda.current_stream(self.device).cuda_stream))

    def set_early(self, params) -> bool:
        """Name the parameters whose gradients are final before the end of backward (the dense heads): step_early()
        updates them on whatever stream is current while the rest of backward runs, step() then only does the others.
        Valid because the update has no cross-parameter term (no clipping: APE_X/Learner.py:123-138).  The early
        parameters must be a contiguous run of the optimizer's list; returns False (and changes nothing) otherwise."""
        idx = sorted(i for i, p in enumerate(self.params) if any(p is q for q in params))
        if not idx or idx != list(range(idx[0], idx[-1] + 1)):
            return False
        self._early = (idx[0], idx[-1] + 1)
        return True

    def step_early(self) -> None:
        lo, hi = self._early
        self._launch(lo, hi, None)
        self._early_done = True

    def step(self, want_norm: bool = True) -> torch.Tensor:
        """Update + zero_grad.  Returns the device scalar sqrt(sum_i ||g_i||_2) (of the pre-step grads)."""
        n = len(self.params)
        if getattr(self, "_early_done", False):
            lo, hi = self._early
            self._early_done = False
            if lo > 0:
                self._launch(0, lo, None)
            if hi < n:
                self._launch(hi, n, None)
            if want_norm:
                check(_lib.load().b2rl_rmsprop_norm_finish(self._scratch.data_ptr(), n, self.grad_norm.data_ptr(),
                                                           torch.cuda.current_stream(self.device).cuda_stream))
            return self.grad_norm
        self._launch(0, n, self.grad_norm.data_ptr() if want_norm else None)
        return self.grad_norm

    def zero_grad(self, set_to_none: bool = False) -> None:
        for p in self.params:
            p.grad.zero_()


def flat_grads(params) -> torch.Tensor:
    """Pre-allocate every .grad as a view into ONE zero buffer, largest tensors first (so equally shaped big matrices —
    the dense heads' first layers — lie back to back and one GEMM can write all of them: linear._stacked_rows).
    Each view keeps its parameter's element order.  Returns the buffer."""
    params = [p for p in params]
    order = sorted(range(len(params)), key=lambda i: -params[i].numel())
    total = sum(p.numel() for p in params)
    flat = torch.zeros((total + 3) // 4 * 4, dtype=params[0].dtype, device=params[0].device)
    off = 0
    for i in order:
        p = params[i]
        p.grad = flat[off:off + p.numel()].as_strided(p.shape, p.stride())
        off += p.numel()
    return flat


def _dense(t: torch.Tensor) -> bool:
    """True if t's storage is a dense permutation (contiguous in some dim order)."""
    return t.is_contiguous() or t.is_contiguous(memory_format=torch.channels_last) or \
        (t.numel() == t.untyped_storage().nbytes() // t.element_size())
