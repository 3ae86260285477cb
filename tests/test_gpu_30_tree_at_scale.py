"""The sum-tree bit for bit against the binary tree at the capacities the learners run.

DESIGN.md §0 promises that the sparse radix-16 sum-tree (csrc/tree.cu) holds, and descends through, exactly the values
of the binary tree over the same leaves (baseline/sumtree.py, restated as oracle.SumTreeOracle).  tree.cu picks its code
path by capacity: the build runs in one launch up to 296 CTAs and in two from cap2 = 2^21 on, the small update keeps
stored level `ks` (the first with at most 4096 nodes) in shared memory, the large update launches per level up to level
`kt` (the first with at most 256 nodes) and a narrower top group spans 1 to 3 binary levels.  Each capacity below selects
a different mix of them; together they reach every branch.

One scenario runs at every capacity: a build shaped like a live replay, small and large scattered updates, ring pushes,
pipelined retirements and evictions around the end of the ring, and a second, all-dyadic build for draws that land
exactly on leaf boundaries.  After every step every stored level (fp64 sums, fp32 minima) and the leaves are compared
with the oracle bit for bit, and 4096 draws with explicit uniforms must return the oracle's slots and probabilities bit
for bit (IS weights to 2 ulp, a pow is involved)."""
import gc
import math
import os
import time

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BETA = 0.4
DRAWS = 4096
F32, F64 = np.float32, np.float64

# capacity -> what tree_shape() must report (cap2, G, top_bits), and what that selects in tree.cu
SCALES = [
    # capacity          cap2     G  top   small update ks (level-ks nodes) | large update kt | build
    (1 << 20,           1 << 20, 5, 4),  # ks 2 (4096, all of US_SMEM_NODES) | kt 3 | one launch (256 CTAs)
    ((1 << 20) + 1,     1 << 21, 6, 1),  # ks 3 (512)                         | kt 4 | two launches
    (1_999_999,         1 << 21, 6, 1),  # as above; the ring's end lies inside a 16-leaf group
    ((1 << 22) + 12345, 1 << 23, 6, 3),  # ks 3 (2048)                        | kt 4 | two launches
    (1 << 24,           1 << 24, 6, 4),  # ks 3 (4096)                        | kt 4 | two launches
    ((1 << 24) + 1,     1 << 25, 7, 1),  # ks 4 (512)                         | kt 5 | two launches
]


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import replay
    return replay


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _host_bytes_available() -> int:
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_AVPHYS_PAGES")


def _live_prios(rng, n):
    """Priorities as a live replay holds them: (|td| clipped to 1 + eps) ** alpha."""
    return ((np.abs(rng.standard_normal(n)).clip(max=1) + 1e-7) ** 0.6).astype(F32)


# --------------------------------------------------------------------------------------------------------------------
# The oracle: SumTreeOracle(cap2) over the leaves of RingModel(capacity).  A node of the binary tree is a pure function
# of the leaves below it, so refreshing only the ancestors of the written slots, or rebuilding every level, gives the
# state SumTreeOracle.update would reach; both are vectorised here (update loops in Python).
# --------------------------------------------------------------------------------------------------------------------
class Model:
    def __init__(self, capacity, cap2):
        self.capacity, self.cap2 = capacity, cap2
        self.T = O.SumTreeOracle(cap2)
        self.M = O.RingModel(capacity)

    def build(self, p):
        n = len(p)
        self.T.build(p)
        self.M.prios[:] = 0
        self.M.prios[:n] = p
        self.M.size, self.M.head = n, n % self.capacity

    def refresh(self, slots):
        """The binary tree after M.prios[slots] changed: leaves, then every ancestor, node = left + right."""
        T, cap2 = self.T, self.cap2
        slots = np.unique(np.asarray(slots, np.int64))
        if slots.size == 0:
            return
        v = self.M.prios[slots]
        T.sum[cap2 + slots] = v.astype(F64)
        T.min[cap2 + slots] = np.where(v > 0, v, F32(np.inf))
        if slots.size * 16 >= cap2:                 # most of the tree: every level, as SumTreeOracle.build does
            lvl = cap2 // 2
            while lvl >= 1:
                T.sum[lvl:2 * lvl] = T.sum[2 * lvl:4 * lvl:2] + T.sum[2 * lvl + 1:4 * lvl:2]
                T.min[lvl:2 * lvl] = np.minimum(T.min[2 * lvl:4 * lvl:2], T.min[2 * lvl + 1:4 * lvl:2])
                lvl //= 2
            return
        i = slots + cap2
        while i[-1] > 1:
            i = np.unique(i >> 1)
            T.sum[i] = T.sum[2 * i] + T.sum[2 * i + 1]
            T.min[i] = np.minimum(T.min[2 * i], T.min[2 * i + 1])

    def update(self, idx, vals):
        """b2rl_tree_update: slots outside [0, capacity) are ignored; of repeated slots the last entry wins (the first
        occurrence in the reversed batch)."""
        idx, vals = np.asarray(idx, np.int64), np.asarray(vals, F32)
        keep = (idx >= 0) & (idx < self.capacity)
        slots, first = np.unique(idx[keep][::-1], return_index=True)
        self.M.prios[slots] = vals[keep][::-1][first]
        self.refresh(slots)

    def push(self, p):
        self.refresh(self.M.push(p))

    def retire(self, n):
        """b2rl_replay_reserve / the retirement of b2rl_replay_ingest_pipelined: the n slots at head read 0, and the
        records they held stop counting once the ring is full."""
        M = self.M
        slots = (M.head + np.arange(n)) % self.capacity
        M.size -= max(0, M.size + n - self.capacity)
        M.prios[slots] = 0
        self.refresh(slots)

    def evict(self, d):
        self.refresh(self.M.evict(d))

    def find(self, u):
        """SumTreeOracle.find for a batch of uniforms (pos = root * u, then `pos < left or right == 0`)."""
        T = self.T
        pos = T.sum[1] * np.asarray(u, F64)
        i = np.ones(pos.shape[0], np.int64)
        for _ in range(self.cap2.bit_length() - 1):
            left = T.sum[2 * i]
            go_left = (pos < left) | (T.sum[2 * i + 1] == 0.0)
            pos = np.where(go_left, pos, pos - left)
            i = 2 * i + (~go_left)
        return i - self.cap2


class Checker:
    """Compares the device tree with the model after every step and counts what it compared."""

    def __init__(self, rep, model, G, rng):
        self.rep, self.S, self.G, self.rng = rep, model, G, rng
        self.steps = self.levels = self.draws = 0

    def levels_match(self, step):
        S, rep, cap2 = self.S, self.rep, self.S.cap2
        bad = []
        leaves = rep.priorities().cpu().numpy()
        diff = np.flatnonzero(leaves.view(np.uint32) != S.M.prios.view(np.uint32))
        if diff.size:
            bad.append(f"  leaves: {diff.size} slots differ, first {diff[:4].tolist()}: device "
                       f"{leaves[diff[:4]].tolist()} oracle {S.M.prios[diff[:4]].tolist()}")
        for k in range(1, self.G + 1):
            sums, mins = rep.tree_level(k)
            sums, mins = sums.cpu().numpy(), mins.cpu().numpy()
            nk = 1 if k == self.G else cap2 >> (4 * k)
            lo = 1 if k == self.G else nk                 # stored level k < G is the heap's row [cap2 >> 4k, 2 * ...)
            want_s, want_m = S.T.sum[lo:lo + nk], S.T.min[lo:lo + nk]
            assert sums.shape == (nk,)
            ds = np.flatnonzero(sums.view(np.uint64) != want_s.view(np.uint64))
            dm = np.flatnonzero(mins.view(np.uint32) != want_m.view(np.uint32))
            for what, d, got, want in (("sums", ds, sums, want_s), ("mins", dm, mins, want_m)):
                if d.size:
                    sh = 4 * k if k < self.G else cap2.bit_length() - 1
                    bad.append(f"  stored level {k} {what}: {d.size} of {nk} nodes differ, first nodes "
                               f"{d[:4].tolist()} (leaves [{d[0] << sh}, {(d[0] + 1) << sh})): device "
                               f"{got[d[:4]].tolist()} oracle {want[d[:4]].tolist()}")
        self.levels += self.G + 1
        assert not bad, f"after {step}: the stored tree differs from the binary tree\n" + "\n".join(bad)

    def draws_match(self, step, u):
        S, rep = self.S, self.rep
        idx, prob, w = rep.sample(len(u), beta=BETA, u01=_dev(u))
        oidx = S.find(u)
        np.testing.assert_array_equal(S.T.sample(u[:32])[0], oidx[:32])   # the batched descent is SumTreeOracle's
        np.testing.assert_array_equal(idx.cpu().numpy(), oidx, err_msg=f"drawn slots after {step}")
        with np.errstate(divide="ignore", over="ignore"):                  # max IS weight +inf: a subnormal minimum
            ow, oprob, omaxw = O.is_weights(S.M.prios[oidx], S.T.total, S.T.min_priority, S.M.size, BETA)
        np.testing.assert_array_equal(prob.cpu().numpy().view(np.uint32), oprob.view(np.uint32),
                                      err_msg=f"probabilities after {step}")
        np.testing.assert_allclose(w.cpu().numpy(), ow, rtol=2.4e-7, err_msg=f"IS weights after {step}")
        st = rep.stats(BETA).cpu().numpy()
        assert st[0] == S.T.total and F32(st[1]) == S.T.min_priority, (step, st, S.T.total, S.T.min_priority)
        np.testing.assert_allclose(st[2], omaxw, rtol=2.4e-7, err_msg=f"max IS weight after {step}")
        self.draws += len(u)
        return idx.cpu().numpy()

    def __call__(self, step):
        assert len(self.rep) == self.S.M.size and self.rep.head == self.S.M.head, step
        self.levels_match(step)
        u = self.rng.random(DRAWS)
        u[0], u[1] = 0.0, 1.0 - 2.0 ** -53
        self.draws_match(step, u)
        self.steps += 1


# --------------------------------------------------------------------------------------------------------------------
# The scenario
# --------------------------------------------------------------------------------------------------------------------
def _live_build(rng, n):
    """Build priorities shaped like a live replay, and the zero slots it holds."""
    p = _live_prios(rng, n)
    d0 = (2 * n) // 3 + 5                               # a region of dyadic priorities, multiples of 2^-12
    p[d0:d0 + 5000] = rng.integers(1, 4097, 5000) * F32(2.0 ** -12)
    z0 = (n // 3) // 256 * 256 - 9                       # mid-group; covers the whole 256-leaf block that starts at z0 + 9
    zero_run = (z0, 16 * 16 + 50)
    p[z0:z0 + zero_run[1]] = 0
    isolated = rng.choice(n, 24, replace=False)
    p[isolated] = 0
    tiny = rng.choice(n, 6, replace=False)              # subnormal and near-underflow priorities: valid (p > 0) slots
    p[tiny] = np.array([2.0 ** -149, 1e-40, 1e-38, 2.0 ** -126, 1e-30, 1e-30], F32)
    return p, zero_run, np.setdiff1d(isolated, tiny), tiny


def _dyadic_build(rng, capacity, zero_run, isolated):
    """All leaves multiples of 2^-12, the same zero slots, and a total that is a power of two, so fp64 prefix sums and
    root * u are exact: u = prefix / total lands exactly on a leaf boundary.  Positive leaves come in pairs of c units
    (c in [4096, 8192)); one adjusting leaf of fewer than P units (P pairs) makes the total 2^m units."""
    p = np.zeros(capacity, F32)
    zero = np.zeros(capacity, bool)
    zero[zero_run[0]:zero_run[0] + zero_run[1]] = True
    zero[isolated] = True
    adj = 5
    zero[adj] = True
    pos = np.flatnonzero(~zero)
    pos = pos[:pos.size // 2 * 2]
    P = pos.size // 2
    m = math.ceil(math.log2(P * 4096))
    c = (1 << m) // P
    k = rng.integers(1, c, P)
    p[pos[0::2]] = k * F32(2.0 ** -12)
    p[pos[1::2]] = (c - k) * F32(2.0 ** -12)
    p[adj] = F32(((1 << m) - P * c) * 2.0 ** -12)
    assert float(p.astype(F64).sum()) == 2.0 ** (m - 12)
    return p


def _scattered(rng, n, capacity, cap2):
    """A write-back batch: random slots with repeats (different values), a few zero priorities and, from 16 entries
    on, slots outside [0, capacity) (a padding leaf among them) that the update must ignore."""
    idx = rng.integers(0, capacity, n)
    if n >= 8:
        again = rng.choice(n, max(1, n // 10), replace=False)
        idx[again] = idx[rng.choice(n, again.size)]
    if n >= 16:
        oob = [-1, capacity, cap2 - 1 if cap2 > capacity else capacity + 1, 1 << 40, -(1 << 40)]
        idx[rng.choice(n, len(oob), replace=False)] = oob
    vals = _live_prios(rng, n)
    vals[rng.random(n) < 0.02] = 0
    return idx, vals


def _run_scenario(R, capacity, cap2, G, top_bits):
    t0 = time.perf_counter()
    rng = np.random.default_rng(capacity)
    # one 4-byte field: the pipelined ingest copies a payload
    rep = R.DeviceReplay(capacity, fields=(R.Field("a", torch.int32, ()),))
    try:
        assert rep.tree_shape() == (cap2, G, top_bits)
        S = Model(capacity, cap2)
        check = Checker(rep, S, G, rng)

        # 1. build: n = capacity - 333 (the ring's head inside a 16-leaf group, empty slots, then the padding)
        n0 = capacity - 333
        p, zero_run, isolated, tiny = _live_build(rng, n0)
        rep.build(_dev(p))
        S.build(p)
        check("build")

        def update(step, idx, vals):
            rep.update(_dev(np.asarray(idx, np.int64)), _dev(np.asarray(vals, F32)))
            S.update(idx, vals)
            check(step)

        # 2. small scattered updates (one CTA, level ks in shared memory)
        update("B = 512 with repeats (bench.py's write-back)", *_scattered(rng, 512, capacity, cap2))
        idx, vals = _scattered(rng, 64, capacity, cap2)
        idx[:3], vals[:3] = tiny[:3], _live_prios(rng, 3)   # the subnormal priorities become ordinary ones
        update("B = 64", idx, vals)
        update("B = 1 at slot 0", [0], _live_prios(rng, 1))
        update("B = 1 at slot capacity - 1", [capacity - 1], _live_prios(rng, 1))
        g16 = np.arange(16) + (n0 // 2) // 16 * 16
        update("a whole 16-leaf group zeroed", g16, np.zeros(16, F32))
        update("the zeroed group refilled", g16, _live_prios(rng, 16))

        # 3. large scattered updates: k_update_level below a level's node count, k_tree_level_all from it on
        level_nodes = [cap2 >> 4 * k for k in range(1, G)]
        for n in [513, 8192] + [m for nk in level_nodes for m in (nk - 1, nk, nk + 1)]:
            update(f"a scattered update of {n}", *_scattered(rng, n, capacity, cap2))

        # 4. ring ranges around the end of the ring
        def push(n):
            pr, head = _live_prios(rng, n), S.M.head
            rep.push([None], torch.from_numpy(pr))
            S.push(pr)
            check(f"push of {n} at head {head}")

        assert S.M.head == capacity - 333
        push(400)                                       # <= 512: the small kernel, wrapping
        push(capacity)                                  # every slot, from the middle of the ring
        push(capacity - S.M.head - 1500)                # head to capacity - 1500
        pin = [(torch.zeros(1000, dtype=torch.int32).pin_memory(),
                torch.from_numpy(_live_prios(rng, 1000)).pin_memory()) for _ in range(2)]
        pending = None
        for b, (x, pr) in enumerate(pin):               # retire [cap - 1500, cap - 500), then publish it and
            rep.ingest_pipelined([x], pr)               # retire [cap - 500, cap) + [0, 500): both segments
            if pending is not None:
                S.push(pending)
            S.retire(1000)
            pending = pr.numpy().copy()
            check(f"pipelined ingest {b}: retirement of 1000")
        rep.ingest_pipelined(None)
        S.push(pending)
        check("pipelined ingest flushed: the wrapped batch published")
        rep.push_begin([None], 1000)
        S.retire(1000)
        check("push_begin: retirement of 1000")
        pr = _live_prios(rng, 1000)
        rep.push_commit(torch.from_numpy(pr))
        S.push(pr)
        check("push_commit of 1000")
        assert (S.M.head, S.M.size) == (1500, capacity)

        def evict(d):
            tail = (S.M.head - S.M.size) % capacity
            rep.evict(d)
            S.evict(d)
            check(f"evict of {d} from tail {tail}")

        evict(capacity - 1650)                          # tail to capacity - 150
        evict(300)                                      # <= 512, wrapping
        push(capacity)                                  # full again, tail = head = 1500
        push(capacity - 2200)                           # tail = head = capacity - 700
        evict(1000)                                     # > 512, wrapping: both segments

        # device-RNG draws never pick an empty slot or one beyond capacity
        def rng_draws(step):
            rep.seed(capacity, 0)
            idx, _, _ = rep.sample(1 << 20)
            i = idx.cpu().numpy()
            assert i.min() >= 0 and i.max() < capacity, step
            assert (S.M.prios[i] > 0).all(), f"{step}: drew slots of priority 0: {np.unique(i[S.M.prios[i] == 0])[:8]}"
            check.draws += 1 << 20

        rng_draws("after the ring operations")

        # 5. edge draws on an all-dyadic build (n = capacity: head 0) with the same zero slots and padding
        p2 = _dyadic_build(rng, capacity, zero_run, isolated)
        rep.build(_dev(p2))
        S.build(p2)
        check("dyadic build")
        total = S.T.total
        assert math.frexp(total)[0] == 0.5, total
        prefix = np.concatenate([[0.0], np.cumsum(p2.astype(F64))])      # exact: integers of 2^-12 below 2^53
        positive = np.flatnonzero(p2 > 0)
        J = np.unique(np.concatenate([
            [0, zero_run[0], positive[-1]], isolated,                   # boundaries in front of the zero slots
            rng.choice(capacity // 16, 64) * 16, rng.choice(capacity // 256, 64) * 256,
            rng.choice(capacity // 4096, 64) * 4096, rng.integers(0, capacity, 256)]))
        J = J[prefix[J] < total]
        u_at = prefix[J] / total                                         # exact: total is a power of two
        u_before = np.nextafter(u_at[u_at > 0], 0.0)
        u = np.concatenate([[0.0, 1.0 - 2.0 ** -53], u_at, u_before])
        got = check.draws_match("edge draws", u)
        # independently of the descent: prefix[j] <= root * u < prefix[j + 1] for a positive leaf j
        first_at_or_after = positive[np.searchsorted(positive, J)]
        last_before = positive[np.searchsorted(positive, J[u_at > 0]) - 1]
        want = np.concatenate([[positive[0], positive[-1]], first_at_or_after, last_before])
        np.testing.assert_array_equal(got, want)
        assert (p2[got] > 0).all()
        rng_draws("on the dyadic build")

        print(f"\ncapacity {capacity}: cap2 2^{cap2.bit_length() - 1}, G {G}, top_bits {top_bits}: {check.steps} steps "
              f"checked, {check.levels} stored levels (leaves included) compared bit for bit, {check.draws} draws, "
              f"{time.perf_counter() - t0:.1f} s")
    finally:
        rep.close()


@pytest.mark.parametrize("capacity,cap2,G,top_bits", SCALES, ids=[str(s[0]) for s in SCALES])
def test_tree_matches_binary_tree_at_scale(R, capacity, cap2, G, top_bits):
    need = 64 * cap2 + (1 << 30)    # oracle fp64 sums + fp32 minima (24 B per leaf), the ring model, read-backs
    if _host_bytes_available() < need:
        pytest.skip(f"the oracle of a {cap2}-leaf tree needs about {need / 1e9:.1f} GB of host memory")
    try:
        _run_scenario(R, capacity, cap2, G, top_bits)
    finally:
        gc.collect()
        torch.cuda.empty_cache()


def test_tree_level_refuses_bad_arguments_and_reads_small_trees(R):
    """b2rl_tree_level on a live handle: a level outside 0..G or a null n_nodes is refused; every stored level of a
    small tree (G = 2, a 3-level top group) equals the binary tree's."""
    import ctypes as C
    from distributed_rl_b200._lib import B2RLError
    rep = R.DeviceReplay(100, fields=())
    try:
        assert rep.tree_shape() == (128, 2, 3)
        for k in (-1, 3, 1 << 20):
            with pytest.raises(B2RLError, match="no such stored level"):
                rep.tree_level(k)
        assert rep.lib.b2rl_tree_level(rep._h, 1, None, None, None, None, None, None) < 0
        assert b"null n_nodes" in rep.lib.b2rl_last_error()
        n = C.c_int64(-1)
        assert rep.lib.b2rl_tree_level(rep._h, 2, C.byref(n), None, None, None, None, None) == 0 and n.value == 1
        sums, mins = rep.tree_level(1)                   # the empty tree: sums 0, minima +inf
        assert (sums.cpu().numpy() == 0).all() and np.isinf(mins.cpu().numpy()).all()
        rng = np.random.default_rng(30)
        p = _live_prios(rng, 100)
        p[[3, 40, 41]] = 0
        rep.build(_dev(p))
        S = Model(100, 128)
        S.build(p)
        Checker(rep, S, 2, rng)("a 100-slot build")
    finally:
        rep.close()
