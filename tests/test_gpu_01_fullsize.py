"""Full-size (BASELINE.json configs[1]/[2]/[3]) checks through size-independent properties —
the oracle cannot hold 59 GB, so the payload is verified against its counter hash, the tree
against fp64 reductions of its own leaves, sampling against chi-square, and updates against
idempotence / last-writer-wins."""
import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if torch.cuda.get_device_properties(0).total_memory < 75e9:
        pytest.skip("needs an 80 GB device (59 GB Ape-X payload)")
    from distributed_rl_b200 import replay
    return replay


def test_apex_2pow20_slots_full_payload(R):
    """C2: 2^20 slots x 56 457 B = 59.2 GB in HBM; batch 512 and 8192."""
    N = 1 << 20
    rep = R.DeviceReplay(N, fields=R.APEX_FIELDS)
    rep.fill_hash(N, seed=0xB200)
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    p = (torch.randn(N, device="cuda", generator=g).abs().clamp(max=1) + 1e-7) ** 0.6
    rep.build(p)
    st = rep.stats(0.4).cpu().numpy()
    leaves = rep.priorities()
    assert torch.equal(leaves, p)                                              # leaves round-trip bit-exact
    np.testing.assert_allclose(st[0], float(p.double().sum()), rtol=1e-12)     # fp64 root == fp64 sum of leaves
    assert np.float32(st[1]) == np.float32(p.min().item())
    # gather: every sampled row equals the counter hash of its slot, both frame fields and the scalars
    for n in (512, 8192):
        idx, prob, w = rep.sample(n)
        i = idx.cpu().numpy()
        assert i.min() >= 0 and i.max() < N
        np.testing.assert_array_equal(prob.cpu().numpy(), p[idx].cpu().numpy() / np.float32(st[0]))   # IEEE fp32 division
        assert float(w.max()) <= 1.0 + 1e-6 and float(w.min()) > 0
        out = rep.gather(idx)
        sub = np.random.default_rng(n).choice(n, size=64, replace=False)       # hash 64 rows on the host
        for fi, f in enumerate(R.APEX_FIELDS):
            want = O.hash_rows(fi, i[sub], f.nbytes, 0xB200)
            got = out[f.name][torch.from_numpy(sub).cuda()].contiguous().view(torch.uint8).reshape(64, -1).cpu().numpy()
            np.testing.assert_array_equal(got, want, err_msg=f.name)
    # proportional sampling at full size: chi-square over 256 equal-count bins of the slot range
    draws = 1 << 22
    idx, _, _ = rep.sample(draws)
    counts = torch.bincount(idx // (N // 256), minlength=256).double().cpu().numpy()
    expect = p.double().view(256, -1).sum(1).cpu().numpy() / st[0] * draws
    chi2 = ((counts - expect) ** 2 / expect).sum()
    assert chi2 < 360.0, chi2          # 255 dof: P(chi2 > 360) ~ 1e-5
    # update: last writer wins + idempotent + root stays the fp64 sum of the leaves
    ui = torch.randint(0, N, (8192,), device="cuda", generator=g)
    ui[-100:] = ui[:100]                                      # duplicates: the later value must win
    uv = torch.rand(8192, device="cuda", generator=g) + 0.01
    rep.update(ui, uv)
    after = rep.priorities()
    rep.update(ui, uv)
    assert torch.equal(after, rep.priorities())
    assert torch.equal(after[ui[-100:]], uv[-100:])
    np.testing.assert_allclose(rep.stats().cpu().numpy()[0], float(after.double().sum()), rtol=1e-12)
    # small-batch path (sorted single-CTA kernel) on the same tree
    rep.update(ui[:512], uv[:512] * 0.5)
    np.testing.assert_allclose(rep.stats().cpu().numpy()[0], float(rep.priorities().double().sum()), rtol=1e-12)
    rep.close()


def test_r2d2_2pow20_sequence_slots_tree_and_long_rows(R):
    """C3: 2^20 sequence slots in the tree; payload pool of 2^10 length-80 sequences (2.3 GB): the
    full 2.4 TB payload cannot exist (SURVEY.md §8d) — the gather of 2.26 MB rows is checked on the pool."""
    N = 1 << 20
    tree = R.DeviceReplay(N, fields=())
    g = torch.Generator(device="cuda"); g.manual_seed(2)
    p = torch.rand(N, device="cuda", generator=g) ** 2 + 1e-6
    tree.build(p)
    idx, prob, w = tree.sample(64)
    np.testing.assert_allclose(tree.stats().cpu().numpy()[0], float(p.double().sum()), rtol=1e-12)
    tree.update(idx, torch.ones(64, device="cuda"))
    assert torch.equal(tree.priorities()[idx], torch.ones(64, device="cuda"))
    tree.close()
    pool = 1 << 10
    fields = R.r2d2_fields(80)
    rep = R.DeviceReplay(pool, fields=fields)
    rep.fill_hash(pool, seed=5)
    rep.build(torch.ones(pool, device="cuda"))
    idx = (idx % pool).contiguous()
    out = rep.gather(idx)
    i = idx.cpu().numpy()
    for fi, f in enumerate(fields):
        want = O.hash_rows(fi, i[:8], f.nbytes, 5)
        got = out[f.name][:8].contiguous().view(torch.uint8).reshape(8, -1).cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg=f.name)
    rep.close()


def test_impala_batch_1024_vtrace_linearity(R):
    """C4: T=20, B=1024.  V-trace is linear in (reward, value, bootstrap) for fixed ratios:
    vtrace(a*x) == a*vtrace(x) and additivity, checked on the device at full batch."""
    T, B = 20, 1024
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    pi = torch.rand(T, B, device="cuda", generator=g) * 0.9 + 0.05
    mu = torch.rand(T, B, device="cuda", generator=g) * 0.85 + 0.05
    mk = lambda: (torch.randn(T, B, device="cuda", generator=g), torch.randn(B, device="cuda", generator=g),
                  torch.randn(T, B, device="cuda", generator=g))
    (v1, b1, r1), (v2, b2, r2) = mk(), mk()
    f = lambda v, b, r: R.vtrace(pi, mu, v, b, r, 0.99, 1.0, 1.0, 1.0)
    vt1, a1 = f(v1, b1, r1); vt2, a2 = f(v2, b2, r2); vts, as_ = f(v1 + v2, b1 + b2, r1 + r2)
    np.testing.assert_allclose(vts.cpu().numpy(), (vt1 + vt2).cpu().numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(as_.cpu().numpy(), (a1 + a2).cpu().numpy(), rtol=1e-4, atol=1e-4)
    vtk, ak = f(2 * v1, 2 * b1, 2 * r1)
    np.testing.assert_allclose(vtk.cpu().numpy(), (2 * vt1).cpu().numpy(), rtol=1e-6, atol=1e-6)   # exact scaling by 2
    np.testing.assert_allclose(ak.cpu().numpy(), (2 * a1).cpu().numpy(), rtol=1e-6, atol=1e-6)
