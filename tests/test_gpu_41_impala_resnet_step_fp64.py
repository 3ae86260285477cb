"""The IMPALA learner step on the residual network (impala.resnet_small_model) against fp64 at the shape
tools/bench_impala_resnet.py measures: B = 1024, T = 20, 21 504 frame stacks, on 2 048 rollouts of flat 4x4 blocks
with sparse noise (exact ties inside the pool windows, and near ties).

A. Every hand-written kernel of one eager step, on the inputs the step gave it: the stem forward over all 21 504 stacks
   (every CTA of the persistent kernel loops over 81 or 82), bit for bit against tests/stem_model.py's restatement and
   within check_stem's bounds; the stem's weight gradient over the 20 480 sequence rows, within one fp32 ulp of the
   restatement and within check_stem_wgrad's bound; the 3 872 -> 256 layer's three forwards, dL/dx and dL/dW
   (check_gemm); V-trace (check_vtrace and oracle.vtrace).
B. The whole eager step against a restatement of it without the library in fp64, fp32 and TF32 (test_gpu_35's
   comparison), chunked over rollouts, with every decision the learner took (ReLUs, and the three max-pools' argmax)
   taken by the restatement too; two negative controls wire a fault into the step and must fail the same comparison.

The bounds are those of tests/fp64_bounds.py; each checker prints its [err/tol] or [err/ref] ratio, and each test its
wall time and peak device memory."""
import copy
import time

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import stem_model as M  # noqa: E402
from fp64_bounds import _gen, check_gemm, check_stem, check_stem_wgrad, check_vtrace  # noqa: E402
from test_gpu_35_secondary_steps_fp64 import (_arms, _close, _Comparison, _learner_masks, _plain,  # noqa: E402
                                              _StepSpies)

F = torch.nn.functional
B, T, N = 1024, 20, 2048
ROLLOUT_CHUNK = 128             # rollouts per chunk of the restatement's pass with grad (2 560 stacks)
# Peak device memory of one test here, measured on an H100 80GB HBM3 (700 W): 65.1 GB to 65.7 GB (the negative control
# through another argmax the highest).
MIN_FREE_GB = 70
# check_gemm's max-relative sanity ratio against cuBLAS fp32 for the 3 872 -> 256 layer's forward over 20 480 rows, on
# the step's own inputs.  Measured on an H100 80GB HBM3 (700 W): 3xTF32 6.5e-6 of max|ref|, cuBLAS fp32 1.1e-6: 5.8x
# (the tensor core reads the lo terms truncated, an error of one sign per product that grows with K = 3 872); every
# element stays within 0.013 of check_gemm's derived bound and TF32 / 20 holds with 3x to spare.  Its dL/dx over the
# same rows: 2.0e-6 against 3.9e-7, 5.1x, within 0.10 of the bound.  8 is test_gpu_22's.
VS_CUBLAS_DENSE = 8


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    free, _ = torch.cuda.mem_get_info()
    if free < MIN_FREE_GB << 30:
        pytest.skip(f"needs about {MIN_FREE_GB} GB of free device memory, {free / 2 ** 30:.1f} GB free")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def R(dev):
    from distributed_rl_b200 import replay
    return replay


@pytest.fixture(scope="module")
def L(dev):
    from distributed_rl_b200 import linear
    return linear


@pytest.fixture(autouse=True)
def _time_and_memory(request):
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        print(f"[time] {request.node.name}: {time.perf_counter() - t0:.1f} s, peak device memory "
              f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GB")
        torch.cuda.empty_cache()


def resnet_learner():
    """The IMPALA learner on resnet_small_model at B = 1024, T = 20 over 2 048 rollouts: the small fields filled as
    test_gpu_22's impala_learner fills them, the frames flat 4x4 blocks (as tools/bench_impala_resnet.py makes them)
    with 2 % of the pixels replaced by noise."""
    from distributed_rl_b200 import impala
    cfg = impala.ImpalaConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, UNROLL_STEP=T, LEARNER_DEVICE="cuda:0",
                              MODEL=impala.resnet_small_model())
    torch.manual_seed(0)
    lrn = impala.Learner(cfg, start_replay=False)
    st = lrn._memory.store
    g = _gen(0xB209)
    st.fill_hash(N, seed=0xB205)
    state = st.field_view("state").view(N, T + 1, 4, 84, 84)
    for a in range(0, N, 256):
        blocks = torch.randint(0, 256, (256, T + 1, 4, 21, 21), dtype=torch.uint8, device="cuda", generator=g)
        f = blocks.repeat_interleave(4, dim=3).repeat_interleave(4, dim=4)
        noise = torch.randint(0, 256, f.shape, dtype=torch.uint8, device="cuda", generator=g)
        state[a:a + 256] = torch.where(torch.rand(f.shape, device="cuda", generator=g) < 0.02, noise, f)
    st.field_view("action").copy_(torch.randint(0, 6, (N, T), device="cuda", generator=g, dtype=torch.int32))
    st.field_view("mu").copy_(torch.rand(N, T, device="cuda", generator=g) * 0.85 + 0.05)
    st.field_view("reward").copy_(torch.randn(N, T, device="cuda", generator=g))
    st.field_view("done").copy_((torch.rand(N, device="cuda", generator=g) > 0.05).float())
    st.build(torch.ones(N, device="cuda"))
    return lrn


class _ResnetSpies(_StepSpies):
    """test_gpu_35's step spies plus the stem: the weights each StemPack was packed from, stem_fused's inputs and
    outputs, stem_wgrad's inputs, the gradient it accumulated into (`base`, copied before the call) and its result;
    and the argmax of pool_2 and pool_3 in the learner's pass with grad (max_pool2d's flat indices, as int32)."""

    def __init__(self, monkeypatch, R, L, lrn):
        super().__init__(monkeypatch, R, L, lrn, lrn._memory, "draw")
        self.calls.update(stem_fused=[], stem_wgrad=[])
        self.pool_idx = {}
        orig_pack, orig_fused, orig_wgrad = R.StemPack.pack, R.stem_fused, R.stem_wgrad

        def pack(p, weight):
            self.packed[id(p)] = weight.detach().float().clone()
            return orig_pack(p, weight)

        def stem_fused(frames, idx, p, out=None):
            res = orig_fused(frames, idx, p, out=out)
            self.calls["stem_fused"].append(dict(frames=frames, idx=None if idx is None else idx.clone(),
                                                 weight=self.packed[id(p)], pooled=res[0].clone(),
                                                 argmax=res[1].clone()))
            return res

        def stem_wgrad(frames, idx, gp, argmax, out=None, accumulate=False):
            base = out.clone() if (out is not None and accumulate) else None
            res = orig_wgrad(frames, idx, gp, argmax, out=out, accumulate=accumulate)
            self.calls["stem_wgrad"].append(dict(frames=frames, idx=None if idx is None else idx.clone(),
                                                 gp=gp.detach().clone(), argmax=argmax.clone(), base=base,
                                                 got=res.detach().clone()))
            return res

        for name in ("pool_2", "pool_3"):
            def pool_hook(m, inp, out, name=name):
                if torch.is_grad_enabled():
                    self.pool_idx[name] = F.max_pool2d(inp[0].detach(), 3, 2, 1, return_indices=True)[1].int()
            self.hooks.append(getattr(lrn.model.module00, name).register_forward_hook(pool_hook))

        monkeypatch.setattr(R.StemPack, "pack", pack)
        monkeypatch.setattr(R, "stem_fused", stem_fused)
        monkeypatch.setattr(R, "stem_wgrad", stem_wgrad)


def _resnet_step(R, L, monkeypatch, fault=None):
    """One eager step -> (learner, snapshot of the net before it, spies).  `fault(monkeypatch, learner)` wires a fault
    in after the spies, so the spies record what the kernels computed."""
    lrn = resnet_learner()
    snap = copy.deepcopy(lrn.model)
    spies = _ResnetSpies(monkeypatch, R, L, lrn)
    if fault is not None:
        fault(monkeypatch, lrn)
    lrn.fused_step(use_graph=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    spies.remove_hooks()
    return lrn, snap, spies


# --------------------------------------------------------------------------- #
# A. every kernel of one eager step, on the inputs it received                 #
# --------------------------------------------------------------------------- #
def test_resnet_step_kernels_on_their_inputs(R, L, monkeypatch):
    lrn, _, spies = _resnet_step(R, L, monkeypatch)
    c = spies.calls
    n = {k: len(c[k]) for k in ("stem_fused", "stem_wgrad", "linear3x", "linear3x_backward", "vtrace", "conv1_fused")}
    assert n == dict(stem_fused=1, stem_wgrad=1, linear3x=3, linear3x_backward=1, vtrace=1, conv1_fused=0), n
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    s = c["stem_fused"][0]
    rows = s["idx"]
    assert rows.numel() == (T + 1) * B and s["pooled"].shape == ((T + 1) * B, 16, 42, 42)
    want_p, want_a = M.forward_t(s["frames"], rows, s["weight"])
    bad = ((s["pooled"].view(torch.int32) != want_p.view(torch.int32)) | (s["argmax"] != want_a)).flatten(1).any(1)
    del want_p, want_a
    grid = min(rows.numel(), 2 * sms)
    print(f"[bits] resnet step stem_fused: {int(bad.sum())} of {rows.numel()} stacks differ from the restatement "
          f"(grid {grid}: {rows.numel() // grid} to {-(-rows.numel() // grid)} stacks per CTA)")
    assert not bad.any(), f"stacks {bad.nonzero()[:8, 0].tolist()} differ from the restatement"
    check_stem("resnet step stem_fused", s["frames"], rows, s["weight"], s["pooled"], s["argmax"])

    w = c["stem_wgrad"][0]
    assert torch.equal(w["idx"], rows[:T * B]) and torch.equal(w["argmax"], s["argmax"][:T * B])
    want = M.wgrad_t(w["frames"], w["idx"], w["gp"], w["argmax"], base=w["base"])
    d = M.ulps(w["got"], want)
    print(f"[bits] resnet step stem_wgrad over {T * B} stacks: {int((d > 0).sum())} of {d.numel()} elements one ulp "
          f"from the restatement, {int((d > 1).sum())} further")
    assert d.max().item() <= 1
    check_stem_wgrad("resnet step stem_wgrad", w["frames"], w["idx"], w["gp"], w["argmax"], w["got"], base=w["base"])
    assert torch.equal(spies.grads["module00.conv_1.weight"], w["got"])

    assert [x["x"].shape[0] for x in c["linear3x"]] == [B, T * B, T * B]
    for x in c["linear3x"]:
        assert x["x"].shape[1] == 3872 and x["w"].shape == (256, 3872)
        check_gemm(f"resnet step linear3x M={x['x'].shape[0]}", x["x"], x["w"], x["y"], vs_cublas=VS_CUBLAS_DENSE)
    b = c["linear3x_backward"][0]
    assert b["x"].shape == (T * B, 3872) and b["gw"] is not None
    check_gemm("resnet step dense dL/dx", b["gy"], b["w"].T.contiguous(), b["gx"], vs_cublas=VS_CUBLAS_DENSE)
    check_gemm("resnet step dense dL/dW", b["gy"].T.contiguous(), b["x"].T.contiguous(), b["gw"])
    assert torch.equal(spies.grads["module01.MLP_1.weight"], b["gw"])

    v = c["vtrace"][0]
    pi, mu, value, boot, rew, gamma, lam, cbar, pbar = v["args"]
    assert pi.shape == (T, B)
    check_vtrace("resnet step vtrace", pi, mu, value, boot, rew, gamma, lam, cbar, pbar, v["vt"], v["adv"])
    ovt, oadv, _ = O.vtrace(*(x.cpu().numpy() for x in (pi, mu, value, boot, rew)), gamma, lam, cbar, pbar)
    np.testing.assert_allclose(v["vt"].cpu().numpy(), ovt, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(v["adv"].cpu().numpy(), oadv, rtol=1e-5, atol=1e-5)
    _close(lrn)


# --------------------------------------------------------------------------- #
# B. the whole step against an fp64 restatement                                #
# --------------------------------------------------------------------------- #
class _ChunkRows:
    """A decision of the learner's pass with grad, (T, B, ...) time-major, read at the rollouts of the restatement's
    current chunk (`cur` = [b0, b1]) as that chunk's time-major rows: what _learner_masks multiplies by."""

    def __init__(self, full, cur):
        self.full, self.cur = full, cur

    def to(self, dtype):
        b0, b1 = self.cur
        return self.full[:, b0:b1].reshape(-1, *self.full.shape[2:]).to(dtype)


def _stem_positions(argmax, W=84):
    """The stem's argmax (3i + j of each window) as max_pool2d's flat index into the conv output."""
    a = argmax.long()
    PH, PW = a.shape[-2:]
    py = torch.arange(PH, device=a.device).view(PH, 1)
    px = torch.arange(PW, device=a.device).view(1, PW)
    return (2 * py - 1 + a // 3) * W + (2 * px - 1 + a % 3)


def _resnet_compare(lrn, snap, spies):
    """pi_a, value, boot, objActor, criticLoss and every pre-clip gradient against the restatement: the drawn rollouts
    read from the store, the bootstrap stacks without grad, then the sequence stacks with grad one chunk of rollouts at
    a time.  The loss is a mean of per-row terms formed from the learner's own vt and adv, so each chunk adds its rows'
    sum over T B and the chunks' gradients add up.  In the pass with grad every ReLU takes the learner's decision
    (_learner_masks), pool_1 takes the stem kernel's argmax and pool_2, pool_3 the indices of the learner's own
    max_pool2d: an element within rounding of a tie flips between precisions, and one flip moves a whole gradient term."""
    c, cfg = spies.calls, lrn.cfg
    A = cfg.ACTION_SIZE
    idx = c["draw"][0]
    st = lrn._memory.store
    f = {k: st.field_view(k)[idx] for k in ("state", "action", "mu", "reward", "done")}
    pi, mu, value, boot, rew = c["vtrace"][0]["args"][:5]
    vt, adv = c["vtrace"][0]["vt"], c["vtrace"][0]["adv"]
    assert torch.equal(mu, f["mu"].t()) and torch.equal(rew, f["reward"].t())
    action = f["action"].long().t()                                 # (T, B)
    frames = f["state"].view(B, T + 1, 4, 84, 84)
    cur = [0, 0]
    masks = {k: _ChunkRows(m.view(T, B, *m.shape[1:]), cur) for k, m in spies.masks.items()}
    pools = {"pool_1": c["stem_fused"][0]["argmax"][:T * B].view(T, B, 16, 42, 42)}
    pools.update({k: v.view(T, B, *v.shape[1:]) for k, v in spies.pool_idx.items()})

    def restate(dtype):
        m = _learner_masks(_plain(snap, dtype), masks)
        for name, ind in pools.items():
            def pool_hook(mod, inp, out, name=name, ind=ind):
                if torch.is_grad_enabled():
                    b0, b1 = cur
                    at = ind[:, b0:b1].reshape(-1, *ind.shape[2:])
                    at = _stem_positions(at) if name == "pool_1" else at.long()
                    return inp[0].flatten(2).gather(2, at.flatten(2)).view_as(out)
            getattr(m.module00, name).register_forward_hook(pool_hook)
        with torch.no_grad():
            out_last = m.forward([frames[:, T].to(dtype) / 255.0])[0]
        pi_a, val = torch.empty(T, B, dtype=dtype, device="cuda"), torch.empty(T, B, dtype=dtype, device="cuda")
        obj, critic = 0.0, 0.0
        for b0 in range(0, B, ROLLOUT_CHUNK):
            b1 = min(B, b0 + ROLLOUT_CHUNK)
            cur[:] = [b0, b1]
            x = frames[b0:b1, :T].transpose(0, 1).reshape(-1, 4, 84, 84).to(dtype) / 255.0   # time-major rows
            out = m.forward([x])[0]
            del x
            logits = out[:, :A]
            logp = torch.log_softmax(logits, dim=-1)
            entropy = -(logp.exp() * logp).sum(-1, keepdim=True)
            act = action[:, b0:b1].reshape(-1, 1)
            o = (logp.gather(1, act) * adv[:, b0:b1].to(dtype).reshape(-1, 1) + cfg.ENTROPY_R * entropy).sum() / (T * B)
            k = (out[:, -1] - vt[:, b0:b1].to(dtype).reshape(-1)).pow(2).sum() / (2 * T * B)
            (-o + k).backward()
            obj, critic = obj + o.detach(), critic + k.detach()
            pi_a[:, b0:b1] = torch.softmax(logits.detach(), dim=-1).gather(1, act)[:, 0].view(T, b1 - b0)
            val[:, b0:b1] = out[:, -1].detach().view(T, b1 - b0)
            del out, logits, logp, entropy
        return dict(pi_a=pi_a, value=val, boot=out_last[:, -1] * f["done"].to(dtype), objActor=obj,
                    criticLoss=critic, grads={n: p.grad for n, p in m.named_parameters()})

    cmp = _Comparison("IMPALA resnet", _arms(restate))
    for key, got in (("pi_a", pi), ("value", value), ("boot", boot)):
        cmp(key, got)
    # Means over 20 480 terms, in which TF32's roundings average out (as in test_gpu_35): the fp32 criterion alone.
    for key in ("objActor", "criticLoss"):
        cmp(key, lrn.last[key], sharp=False)
    for name, g in spies.grads.items():
        cmp(f"dL/d {name}", g, lambda arm, key: arm["grads"][key[5:]], k=_grad_k(name), sharp=name not in UNSHARP)
    cmp.check()


# Measured on an H100 80GB HBM3 (700 W), max|err| / max|ref64| of the learner's pre-clip gradients against the fp64 arm,
# and its ratio to the fp32 arm's:
#  - conv_1 (the stem's kernel) and section 1's residual blocks: 4.8x and 2.5x to 4.3x, within the default k = 16.
#    Those blocks' gradients sum 20 480 x 42 x 42 terms that largely cancel: even the fp32 arm errs 4.2e-5 to 8.3e-5,
#    only 6x to 22x below TF32's 4.8e-4 to 1.2e-3, so the TF32 criterion cannot hold for them (sharp=False).
#  - conv_2, conv_3, sections 2 and 3 and the 3 872 -> 256 layer: 1.9e-5 to 3.1e-5, 11x to 27x the fp32 arm and 25x
#    to 59x below TF32, except block_3_1.conv_1: 2.5e-5 against TF32's 4.8e-4, 19x (sharp=False for it alone).  The
#    error is the 3xTF32 GEMM's (see VS_CUBLAS_DENSE): h = relu(feat) W1^T errs 5.8x cuBLAS fp32's, and every gradient
#    below the layer is formed from h and from its dL/dx GEMM: k = 32.
#  - the 256 -> 7 layer contracts relu(h) over 20 480 rows: 6.5e-5, 50x to 59x the fp32 arm and 12x below TF32's
#    8.1e-4 (test_gpu_35's 2 592 -> 256 network: 21x and 24x): k = 64, sharp=False.
# The two negative controls below fail at 2.7e5x and 3.4e5x the fp32 arm.
UNSHARP = ({f"module00.block_1_{j}.conv_{i}.weight" for i in (1, 2) for j in (1, 2)}
           | {"module00.block_3_1.conv_1.weight", "module01.MLP_2.weight"})


def _grad_k(name):
    if name == "module01.MLP_2.weight":
        return 64
    if name == "module00.conv_1.weight" or name.startswith("module00.block_1_"):
        return 16
    return 32


def test_resnet_step_against_fp64(R, L, monkeypatch):
    lrn, snap, spies = _resnet_step(R, L, monkeypatch)
    _resnet_compare(lrn, snap, spies)
    _close(lrn)


def test_resnet_comparison_sees_the_bootstrap_one_step_early(R, L, monkeypatch):
    """Negative control: the stem's bootstrap block (the last B rows of its output) replaced by time step T - 1's."""
    def fault(mp, lrn):
        fused = R.stem_fused

        def boot_one_step_early(*a, **k):
            p, am = fused(*a, **k)
            p[T * B:].copy_(p[(T - 1) * B:T * B])
            am[T * B:].copy_(am[(T - 1) * B:T * B])
            return p, am
        mp.setattr(R, "stem_fused", boot_one_step_early)

    lrn, snap, spies = _resnet_step(R, L, monkeypatch, fault)
    with pytest.raises(AssertionError, match="boot"):
        _resnet_compare(lrn, snap, spies)
    _close(lrn)


def test_resnet_comparison_sees_the_stem_gradient_through_another_argmax(R, L, monkeypatch):
    """Negative control: StemGathered handed the stem's argmax rolled by B rows (time step t - 1's windows), so the
    weight gradient folds the pooled gradient into the wrong positions."""
    from distributed_rl_b200 import impala

    def fault(mp, lrn):
        gathered = impala.StemGathered

        class Rolled:
            @staticmethod
            def apply(w, frames, rows, pooled, argmax):
                return gathered.apply(w, frames, rows, pooled, argmax.roll(B, 0))
        mp.setattr(impala, "StemGathered", Rolled)

    lrn, snap, spies = _resnet_step(R, L, monkeypatch, fault)
    with pytest.raises(AssertionError, match=r"dL/d module00\.conv_1\.weight"):
        _resnet_compare(lrn, snap, spies)
    _close(lrn)
