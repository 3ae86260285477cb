"""The sensitivity of the two whole-step checkers of tests/fp64_bounds.py, on the CPU: check_vtrace passes the fp32
numpy oracle's V-trace and fails four mis-wired restatements of it; check_vs_reference passes fp32-rounded data and
rejects TF32-rounded data."""
import numpy as np
import pytest

from oracle import oracle as O

torch = pytest.importorskip("torch")

from fp64_bounds import check_vs_reference, check_vtrace, vtrace_inputs  # noqa: E402

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
