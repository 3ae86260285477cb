"""CPU checks of the stand-alone replay mode for IMPALA: the uniform draw without replacement (its numpy restatement,
tests/uniform_oracle.py), the IMPALA record kind the servers and clients take from an ImpalaConfig, the refusal of the
Redis-protocol pair, and the time-major slot layout and views at the cfg batch (32) and the C4 batch (1024)."""
import pickle

import numpy as np
import pytest

from fake_redis import FakeRedis
from uniform_oracle import feistel_width, philox4x32_10, uniform_draw


@pytest.fixture(scope="module")
def rs():
    from distributed_rl_b200 import build
    build.build()
    from distributed_rl_b200 import replay_server
    return replay_server


def test_the_philox_block_is_the_generator_of_the_sum_tree_draws():
    from oracle.oracle import philox_u01
    for seed, ctr in ((0, 0), (7, 123), (0xFFFF_FFFF_1234, 2 ** 40 + 5)):
        w = philox4x32_10(seed, ctr).astype(np.uint64)
        x = (w[1] << np.uint64(32)) | w[0]
        u = float(x & np.uint64((1 << 53) - 1)) / 2.0 ** 53
        assert u == philox_u01(seed, ctr, 1)[0]


def test_feistel_width_is_the_smallest_even_width_covering_size():
    assert [feistel_width(s) for s in (1, 2, 4, 5, 16, 17, 1000, 1024, 1025, 10000)] == [2, 2, 2, 4, 4, 6, 10, 10, 12, 14]


@pytest.mark.parametrize("n", [1, 16, 32, 60])
def test_draws_are_distinct_and_in_the_valid_region_of_a_wrapped_ring(n):
    from oracle.oracle import RingModel
    ring = RingModel(64)
    for _ in range(10):
        ring.push(np.ones(10))                           # 100 pushes: head 36, full
    ring.evict(3)                                        # size 61, tail 39: the region wraps past the end
    valid = set(((ring.head - ring.size) % 64 + np.arange(ring.size)) % 64)
    for offset in (0, 5, 2 ** 33):
        idx = uniform_draw(11, offset, n, ring.size, 64, ring.head)
        assert len(set(idx.tolist())) == n
        assert set(idx.tolist()) <= valid
    assert not np.array_equal(uniform_draw(11, 0, n, ring.size, 64, ring.head),
                              uniform_draw(11, n, n, ring.size, 64, ring.head)) or n == 1


@pytest.mark.parametrize("size", [1, 3, 16, 61, 1000])
def test_a_draw_of_the_whole_region_is_a_permutation_of_it(size):
    cap, head = 1024, 37
    idx = uniform_draw(3, 99, size, size, cap, head)
    assert sorted(idx.tolist()) == sorted(((head - size) % cap + np.arange(size)) % cap)


def test_more_draws_than_records_raise():
    with pytest.raises(ValueError, match="larger than population"):
        uniform_draw(0, 0, 65, 64, 64, 0)


def test_marginal_counts_are_uniform():
    """4000 fills of 32 draws from 1000 records (not a power of two: the cycle-walk runs): chi-square of the counts."""
    from scipy import stats
    counts = np.zeros(1000, np.int64)
    for f in range(4000):
        np.add.at(counts, uniform_draw(5, 32 * f, 32, 1000, 1000, 0), 1)
    chi2 = ((counts - 128.0) ** 2 / 128.0).sum()
    assert stats.chi2.sf(chi2, 999) > 1e-4


def test_impala_config_maps_to_the_uniform_time_major_kind(rs):
    from distributed_rl_b200 import apex, impala, r2d2
    from distributed_rl_b200 import replay as R
    k = rs.record_kind(impala.ImpalaConfig(UNROLL_STEP=5))
    assert k is rs.KINDS["impala"] and k.replay is impala.Replay
    assert k.list_key == "trajectory" and not k.prioritized and k.steps(impala.ImpalaConfig(UNROLL_STEP=5)) == 5
    assert k.fields(impala.ImpalaConfig(UNROLL_STEP=5)) == R.impala_fields(5)
    assert k.batch({"state": "s", "action": "a", "mu": "mu", "reward": "r", "done": "d"}, "w", "i") == \
        ("s", "a", "mu", "r", "d")
    for cfg in (apex.ApexConfig(), r2d2.R2D2Config()):
        kk = rs.record_kind(cfg)
        assert kk.prioritized and kk.list_key == "experience"


def test_the_redis_protocol_pair_refuses_an_impala_config(rs):
    from distributed_rl_b200 import impala
    cfg = impala.ImpalaConfig(LEARNER_DEVICE="cpu")
    with pytest.raises(ValueError, match="no impala mode"):
        rs.ReplayServer(cfg, FakeRedis())
    with pytest.raises(ValueError, match="no impala mode"):
        rs.Replay_Server(cfg, FakeRedis())


def _align(x, a):
    return (x + a - 1) // a * a


def _client(rs, cfg, batch):
    """A DeviceReplayClient without a server: only its layout, fields and kind (what _views and update read)."""
    class _Ring:
        layout = rs.serve_layout(batch, 2, [f.nbytes for f in rs.record_kind(cfg).fields(cfg)])
    c = rs.DeviceReplayClient.__new__(rs.DeviceReplayClient)
    c.cfg, c.kind, c.ring = cfg, rs.record_kind(cfg), _Ring()
    c.fields = c.kind.fields(cfg)
    return c


@pytest.mark.parametrize("batch", [32, 1024])
def test_time_major_slot_layout_and_views(rs, batch):
    """(T+1) x 28224-byte frame rows, T-word action / mu / reward, done fp32: the bytes per field of a batch-major
    slot; the views are s (T+1, B, 28224), a / mu / r (T, B), done (B,), each a view of the slot buffer."""
    import torch
    from distributed_rl_b200 import impala
    T = 20
    cfg = impala.ImpalaConfig(BATCHSIZE=batch, UNROLL_STEP=T, LEARNER_DEVICE="cpu")
    c = _client(rs, cfg, batch)
    L = c.ring.layout
    fb = [f.nbytes for f in c.fields]
    assert fb == [21 * 28224, 80, 80, 80, 4]
    off = _align(16 + 8 * batch + 4 * batch, 16)
    want = []
    for b in fb:
        want.append(off)
        off = _align(off + b * batch, 16)
    assert [L.field_off[i] for i in range(5)] == want
    assert L.slot_bytes == _align(off, 128)
    if batch == 1024:
        assert L.field_off[1] - L.field_off[0] == 606_928_896            # the 607 MB frame table of a C4 minibatch
    buf = torch.empty(L.slot_bytes, dtype=torch.uint8)
    header, idx, w, b = c._views(buf)
    s, a, mu, r, d = c.kind.batch(b, w, idx)
    assert s.shape == (T + 1, batch, 28224) and s.dtype == torch.uint8 and s.is_contiguous()
    assert s.data_ptr() == buf.data_ptr() + L.field_off[0]
    assert s.view((T + 1) * batch, 4, 84, 84).data_ptr() == s.data_ptr()     # conv_1's frame table, no copy
    for t, i, dt in ((a, 1, torch.int32), (mu, 2, torch.float32), (r, 3, torch.float32)):
        assert t.shape == (T, batch) and t.dtype == dt and t.data_ptr() == buf.data_ptr() + L.field_off[i]
    assert d.shape == (batch,) and d.dtype == torch.float32 and d.data_ptr() == buf.data_ptr() + L.field_off[4]
    assert idx.shape == (batch,)


def test_the_client_posts_no_write_back_for_the_uniform_kind(rs):
    import torch
    from distributed_rl_b200 import impala
    c = _client(rs, impala.ImpalaConfig(LEARNER_DEVICE="cpu"), 32)
    with pytest.raises(TypeError, match="no priorities"):
        c.update(torch.arange(4), torch.ones(4))


def test_the_server_publishes_no_is_weight_for_the_uniform_kind(rs):
    """ImpalaConfig has no BETA and the store's sum-tree holds unit priorities: SERVE_STATS carries a max weight of 0,
    without reading cfg.BETA or calling store.stats()."""
    from distributed_rl_b200 import impala

    class _Store:
        def __len__(self):
            return 123

        def stats(self, beta):
            raise AssertionError("stats() of a uniform replay")
    srv = rs.DeviceReplayServer.__new__(rs.DeviceReplayServer)
    srv.cfg, srv.kind, srv.store = impala.ImpalaConfig(LEARNER_DEVICE="cpu"), rs.KINDS["impala"], _Store()
    srv.connect, srv._stats_t = FakeRedis(), 0.0
    srv._publish_stats(True)
    assert pickle.loads(srv.connect.get(rs.STATS_KEY)) == (123, 0.0)
    m = rs.ServedMemory(srv.connect)
    assert len(m) == 123 and m.max_weight == 0.0


def test_the_server_waits_for_a_batch_of_records_before_a_uniform_fill(rs):
    from distributed_rl_b200 import apex, impala

    class _Store:
        def __init__(self, n):
            self.n = n

        def __len__(self):
            return self.n
    srv = rs.DeviceReplayServer.__new__(rs.DeviceReplayServer)
    srv.cfg, srv.kind = impala.ImpalaConfig(BATCHSIZE=32, BUFFER_SIZE=8, LEARNER_DEVICE="cpu"), rs.KINDS["impala"]
    for n, ok in ((8, False), (20, False), (32, True)):
        srv.store = _Store(n)
        assert srv._can_fill() is ok
    srv.cfg, srv.kind, srv.store = apex.ApexConfig(BATCHSIZE=32, BUFFER_SIZE=8), rs.KINDS["apex"], _Store(20)
    assert srv._can_fill()                              # a draw with replacement needs no more than BUFFER_SIZE
