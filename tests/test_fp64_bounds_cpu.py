"""The sensitivity of checkers of tests/fp64_bounds.py, on the CPU: check_vtrace passes the fp32 numpy oracle's V-trace
and fails four mis-wired restatements of it; check_vs_reference passes fp32-rounded data and rejects TF32-rounded data;
check_stem and check_stem_wgrad pass the stem's exact arithmetic (tests/stem_model.py) on adversarial stacks and fail
four mutants of it."""
import numpy as np
import pytest

from oracle import oracle as O

torch = pytest.importorskip("torch")

import stem_model as M  # noqa: E402
from fp64_bounds import check_stem, check_stem_wgrad, check_vs_reference, check_vtrace, vtrace_inputs  # noqa: E402

F32 = np.float32
GAMMA = 0.99


def _vtrace32(pi_a, mu_a, value, boot, reward, gamma, c_lambda, c_bar, p_bar, mutant=None):
    """oracle.vtrace's arithmetic, op for op, with one deliberate fault when `mutant` is set."""
    g = F32(gamma)
    ratio = np.exp((np.log(pi_a) - np.log(mu_a)).astype(F32)).astype(F32)
    T, B = value.shape
    if mutant == "bootstrap one step early":
        boot = value[T - 1]
    vmt = np.zeros((T, B), F32)
    for i in reversed(range(T)):
        if i == T - 1:
            vmt[i] = ((reward[i] + (g * boot).astype(F32)).astype(F32) - value[i]).astype(F32)
            continue
        td = ((reward[i] + (g * value[i + 1]).astype(F32)).astype(F32) - value[i]).astype(F32)
        cr = {"clip dropped": ratio[i], "p_bar for c_bar": np.minimum(F32(p_bar), ratio[i])}.get(
            mutant, np.minimum(F32(c_bar), ratio[i]))
        cs = (F32(c_lambda) * cr).astype(F32)
        if mutant == "lambda on td":
            td = (F32(c_lambda) * td).astype(F32)
        vmt[i] = ((td * cr).astype(F32) + ((g * cs).astype(F32) * vmt[i + 1]).astype(F32)).astype(F32)
    vtarget = (value + vmt).astype(F32)
    nxt = np.concatenate([vtarget[1:], boot[None, :]], 0)
    atarget = (reward + (g * nxt).astype(F32)).astype(F32)
    adv = ((atarget - value).astype(F32) * np.minimum(F32(p_bar), ratio)).astype(F32)
    return vtarget, adv


def _check(pi, mu, v, boot, r, lam, cbar, pbar, vt, adv):
    t = [torch.from_numpy(np.ascontiguousarray(x)) for x in (pi, mu, v, boot, r, vt, adv)]
    return check_vtrace("fp32 V-trace", *t[:5], GAMMA, lam, cbar, pbar, *t[5:])


@pytest.mark.parametrize("T,B,lam,cbar,pbar", [(20, 256, 0.95, 1.0, 2.0), (100, 7, 1.0, 0.5, 1.0),
                                               (20, 129, 0.95, 2.0, 0.5), (1, 1, 1.0, 1.0, 1.0)])
def test_oracle_vtrace_passes_check_vtrace(T, B, lam, cbar, pbar):
    pi, mu, v, boot, r = vtrace_inputs(T, B, T * 1000 + B)
    vt, adv, _ = O.vtrace(pi, mu, v, boot, r, GAMMA, lam, cbar, pbar)
    mvt, madv = _vtrace32(pi, mu, v, boot, r, GAMMA, lam, cbar, pbar)
    assert np.array_equal(vt, mvt) and np.array_equal(adv, madv)          # the mutants' base is the oracle itself
    _check(pi, mu, v, boot, r, lam, cbar, pbar, vt, adv)


@pytest.mark.parametrize("mutant", ["lambda on td", "clip dropped", "p_bar for c_bar", "bootstrap one step early"])
def test_mutated_vtrace_fails_check_vtrace(mutant):
    T, B, lam, cbar, pbar = 20, 256, 0.95, 1.0, 2.0
    pi, mu, v, boot, r = vtrace_inputs(T, B, 7)
    vt, adv = _vtrace32(pi, mu, v, boot, r, GAMMA, lam, cbar, pbar, mutant=mutant)
    with pytest.raises(AssertionError):
        _check(pi, mu, v, boot, r, lam, cbar, pbar, vt, adv)


def _tf32(x):
    """fp32 -> TF32 (10 mantissa bits), round to nearest."""
    i = x.float().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def test_check_vs_reference_tells_fp32_from_tf32():
    g = torch.Generator().manual_seed(5)
    ref64 = torch.randn(4096, dtype=torch.float64, generator=g) * torch.logspace(-3, 3, 4096, dtype=torch.float64)
    ref32 = ref64.float()
    reftf32 = _tf32(ref32)
    e, e32, etf = check_vs_reference("fp32-rounded", ref64.float(), ref64, ref32, reftf32)
    assert e == e32 and etf > 1000 * e32
    with pytest.raises(AssertionError):
        check_vs_reference("TF32-rounded", reftf32, ref64, ref32, reftf32)
    with pytest.raises(AssertionError):         # 20x fp32's error: above k = 16 and the floor
        check_vs_reference("20 x fp32", ref64 + 20 * (ref32.double() - ref64) + 2e-6 * ref64.abs().max(), ref64,
                           ref32, reftf32)


def _stem_case(n=6, seed=11):
    """Adversarial stem inputs at 84 x 84: frames of 255, of 0, flat 4x4 blocks and random; weights with one dominant
    tap per channel (the others live in the low digits) and an all-zero channel; pooled gradients spanning 30 binades,
    of both signs and of one sign; one stack of positive gradients 21 to 22 binades below its largest, 1, whose digit
    scale is then 2^-4: below half of gy's third digit (2^-20), so that gy rounded one digit coarser loses every one of
    them and the errors cannot cancel; one stack 1e-3 smaller and one so small that its digit exponent clamps at 27."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, size=(n, 4, 84, 84), dtype=np.uint8)
    f[0], f[1] = 255, 0
    f[2] = np.repeat(np.repeat(rng.integers(0, 256, size=(4, 21, 21), dtype=np.uint8), 4, axis=1), 4, axis=2)
    w = (rng.standard_normal((16, 4, 3, 3)) * 0.01).astype(F32)
    for c in range(16):
        w[c, c % 4, c % 3, (c // 4) % 3] = 1.5 if c % 2 else -0.7
    w[9] = 0.0
    g = rng.standard_normal((n, 16, 42, 42)) * np.exp2(-rng.uniform(0, 30, size=(n, 16, 42, 42)))
    g[1] = np.abs(g[1])
    g[5] = np.exp2(-rng.uniform(21.1, 22, size=(16, 42, 42)))    # below half the last digit but one: see above
    g[5, :, 7, 7] = 1.0
    g[3] *= 1e-3
    g[4] *= 1e-33
    return torch.from_numpy(f), torch.from_numpy(w), torch.from_numpy(g.astype(F32))


def _drop_fourth_window(mp):
    mp.setattr(M, "WINDOWS", M.WINDOWS[:3])


def _coarser_gy(mp):
    digits = M.digits_t
    mp.setattr(M, "digits_t", lambda g, e: torch.round(digits(g, e) / 256) * 256)


def test_the_stem_model_passes_check_stem_and_check_stem_wgrad():
    frames, w, gp = _stem_case()
    idx = torch.tensor([5, 0, 2, 2, 1, 3, 4, 0])
    pooled, amax = M.forward_t(frames, idx, w)
    assert torch.equal(pooled[2], pooled[3]) and (amax[1, :, 1:41, 1:41] == 0).all()    # a repeated row; ties
    check_stem("model", frames, idx, w, pooled, amax)
    g = gp[torch.tensor([0, 1, 2, 3, 4, 5, 1, 3])]
    dw = M.wgrad_t(frames, idx, g, amax)
    assert M.digit_exponent_t(4 * g[4].abs().amax(dim=(1, 2))).max().item() == 27
    check_stem_wgrad("model", frames, idx, g, amax, dw)
    base = dw * -3
    check_stem_wgrad("model accumulated", frames, idx, g, amax, M.wgrad_t(frames, idx, g, amax, base=base), base=base)


@pytest.mark.parametrize("mutant", ["three weight digits", "argmax moved to a neighbour"])
def test_mutated_stem_forward_fails_check_stem(mutant, monkeypatch):
    frames, w, _ = _stem_case()
    if mutant == "three weight digits":
        pack = M.pack

        def three(wt):
            q, scale = pack(wt)
            q[3] = 0
            return q, scale
        monkeypatch.setattr(M, "pack", three)
    pooled, amax = M.forward_t(frames, None, w)
    if mutant == "argmax moved to a neighbour":
        a = amax.long()
        amax = torch.where(a % 3 < 2, a + 1, a - 1).to(torch.uint8)   # one column over, inside the window
        amax[:, :, :, 0] = torch.where(amax[:, :, :, 0] % 3 == 0, amax[:, :, :, 0] + 1, amax[:, :, :, 0])
    with pytest.raises(AssertionError):
        check_stem(mutant, frames, None, w, pooled, amax)


@pytest.mark.parametrize("mutant", ["fold drops the fourth window", "gy one digit coarser"])
def test_mutated_stem_wgrad_fails_check_stem_wgrad(mutant, monkeypatch):
    frames, w, gp = _stem_case()
    _, amax = M.forward_t(frames, None, w)
    {"fold drops the fourth window": _drop_fourth_window, "gy one digit coarser": _coarser_gy}[mutant](monkeypatch)
    dw = M.wgrad_t(frames, None, gp, amax)
    monkeypatch.undo()
    assert not torch.equal(dw, M.wgrad_t(frames, None, gp, amax))
    with pytest.raises(AssertionError):
        check_stem_wgrad(mutant, frames, None, gp, amax, dw)
