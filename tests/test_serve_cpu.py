"""CPU checks of the device serve ring's host side: the layout arithmetic of b2rl_serve_layout_init and the
descriptor handshake (ServerSlots / ClientSlots) over a Redis stand-in with real list semantics.  The device work
of each step is replaced by callbacks that log what would be enqueued, so the order of waits, fills and records
can be checked without a GPU."""
import pickle

import pytest

from fake_redis import FakeRedis


@pytest.fixture(scope="module")
def rs():
    from distributed_rl_b200 import build
    build.build()
    from distributed_rl_b200 import replay_server
    return replay_server


def _align(x, a):
    return (x + a - 1) // a * a


@pytest.mark.parametrize("batch,slots", [(1, 1), (3, 2), (32, 4), (512, 4), (512, 16)])
def test_layout_arithmetic(rs, batch, slots):
    from distributed_rl_b200 import replay as R
    fb = [f.nbytes for f in R.APEX_FIELDS]
    L = rs.serve_layout(batch, slots, fb)
    assert (L.batch, L.slots, L.n_fields) == (batch, slots, len(fb))
    # minibatch slot: header, idx, w, then the fields in order; every array 16-byte aligned, slots 128-byte aligned
    regions = [(0, 16), (L.idx_off, 8 * batch), (L.w_off, 4 * batch)] + \
              [(L.field_off[i], b * batch) for i, b in enumerate(fb)]
    for (a, n), (b, _) in zip(regions, regions[1:]):
        assert b % 16 == 0 and b == _align(a + n, 16)       # packed: next array at the first aligned byte
    assert L.slot_bytes % 128 == 0 and L.slot_bytes == _align(regions[-1][0] + regions[-1][1], 128)
    assert [L.field_bytes[i] for i in range(len(fb))] == fb
    # update slot: header, idx int64[B], prio fp32[B]
    assert L.upd_idx_off == 16 and L.upd_prio_off == _align(16 + 8 * batch, 16)
    assert L.upd_slot_bytes == _align(L.upd_prio_off + 4 * batch, 128)
    assert L.upd_base == slots * L.slot_bytes
    assert L.total_bytes == slots * (L.slot_bytes + L.upd_slot_bytes)
    assert all(x % 16 == 0 for x in (L.idx_off, L.w_off, L.upd_base, *L.field_off[:len(fb)]))


def test_layout_of_the_apex_record_at_b512(rs):
    """Two frame stacks of 28 224 B per transition dominate: 28.9 MB per B = 512 minibatch slot."""
    from distributed_rl_b200 import replay as R
    L = rs.serve_layout(512, 4, [f.nbytes for f in R.APEX_FIELDS])
    assert L.field_off[0] == 16 + 4096 + 2048 and L.field_off[1] == L.field_off[0] + 512 * 28224
    assert L.slot_bytes == _align(L.field_off[4] + 512, 128) == 28_912_256


def test_layout_rejects_bad_geometry(rs):
    from distributed_rl_b200 import _lib
    with pytest.raises(_lib.B2RLError, match="batch"):
        rs.serve_layout(0, 4, [4])
    with pytest.raises(_lib.B2RLError, match="slots"):
        rs.serve_layout(8, 0, [4])
    with pytest.raises(_lib.B2RLError, match="field_bytes"):
        rs.serve_layout(8, 2, [0])


class _Log:
    def __init__(self):
        self.ops = []

    def __call__(self, name):
        return lambda *a: self.ops.append((name,) + a)


def test_descriptors_are_served_in_fill_order_and_carry_seq(rs):
    conn, log = FakeRedis(), _Log()
    srv, cli = rs.ServerSlots(conn, 3, 32), rs.ClientSlots(conn, 3)
    assert srv.fill_free(log("fill")) == 3
    assert log.ops == [("fill", 0, 1), ("fill", 1, 2), ("fill", 2, 3)]
    assert [pickle.loads(d) for d in conn.lrange(rs.BATCH_SLOT, 0, -1)] == [(0, 1, 32), (1, 2, 32), (2, 3, 32)]
    cli.poll()
    assert conn.llen(rs.BATCH_SLOT) == 0
    assert [cli.take(log("copy"))[:2] for _ in range(3)] == [(0, 1), (1, 2), (2, 3)]
    assert cli.take(log("copy")) is None                      # nothing filled: the caller returns False
    assert [pickle.loads(d) for d in conn.lrange(rs.RELEASE_SLOT, 0, -1)] == [(0, 1), (1, 2), (2, 3)]


def test_a_slot_is_not_refilled_before_its_release(rs):
    conn, log = FakeRedis(), _Log()
    srv, cli = rs.ServerSlots(conn, 2, 8), rs.ClientSlots(conn, 2)
    srv.fill_free(log("fill"))
    assert srv.fill_free(log("fill")) == 0 and srv.collect_releases(log("wait")) == 0      # both slots are out
    cli.poll()
    cli.take(log("copy"))                                     # slot 0 released, slot 1 still held by the learner
    assert srv.collect_releases(log("wait")) == 1
    assert srv.fill_free(log("fill")) == 1
    # the server stream waits on released[0] BEFORE slot 0 is filled again; slot 1 is never touched
    assert log.ops[-2:] == [("wait", 0), ("fill", 0, 3)]
    assert srv.free == [] and srv.out == {1: 2, 0: 3}
    cli.poll()
    assert [cli.take(log("copy"))[:2] for _ in range(2)] == [(1, 2), (0, 3)]
    # a release the server did not hand out is refused
    conn.rpush(rs.RELEASE_SLOT, pickle.dumps((1, 99)))
    with pytest.raises(RuntimeError, match="did not hand out"):
        srv.collect_releases(log("wait"))


def test_the_client_posts_its_release_only_after_the_copy(rs):
    conn = FakeRedis()
    srv, cli = rs.ServerSlots(conn, 1, 4), rs.ClientSlots(conn, 1)
    srv.fill_free(lambda k, s: None)
    cli.poll()
    seen = []
    cli.take(lambda k: seen.append(conn.llen(rs.RELEASE_SLOT)))
    assert seen == [0] and conn.llen(rs.RELEASE_SLOT) == 1


def test_update_flow(rs):
    conn, log = FakeRedis(), _Log()
    srv, cli = rs.ServerSlots(conn, 2, 8), rs.ClientSlots(conn, 2)
    assert cli.put_update(log("write"), 8) and cli.put_update(log("write"), 5)
    assert not cli.put_update(log("write"), 3)                 # both update slots are with the server
    assert srv.apply_updates(log("apply")) == 13
    assert log.ops == [("write", 0, 1), ("write", 1, 2), ("apply", 0, 8), ("apply", 1, 5)]
    assert [pickle.loads(d) for d in conn.lrange(rs.UPDATE_DONE, 0, -1)] == [(0, 1), (1, 2)]
    assert not cli.put_update(log("write"), 3)                 # not handed back until the client polls
    cli.poll()
    assert cli.put_update(log("write"), 3) and log.ops[-1] == ("write", 0, 3)
    assert srv.apply_updates(log("apply")) == 3 and srv.apply_updates(log("apply")) == 0


def test_a_learner_start_up_wipe_keeps_the_server_handshake(rs):
    """apex.Learner(connect=..., memory=DeviceReplayClient) wipes stale keys after the client has attached: the
    server's keys (ring, client events, descriptors in flight, actor records) must survive it, stale ones must not."""
    from distributed_rl_b200 import wire
    conn, log = FakeRedis(), _Log()
    srv, cli = rs.ServerSlots(conn, 2, 8), rs.ClientSlots(conn, 2)
    conn.set(rs.RING_KEY, b"ring"); conn.set(rs.CLIENT_KEY, b"events"); conn.rpush("experience", b"rec")
    conn.set("Start", b"stale"); conn.set(b"state_dict", b"stale")
    srv.fill_free(log("fill"))                                 # two BATCH_SLOT descriptors in flight
    assert rs.DeviceReplayClient.KEEP_KEYS == rs.SERVER_KEYS
    assert wire.wipe_stale_keys(conn, keep=rs.DeviceReplayClient.KEEP_KEYS) == 2
    assert conn.get("Start") is None and conn.get(b"state_dict") is None
    assert conn.get(rs.RING_KEY) == b"ring" and conn.get(rs.CLIENT_KEY) == b"events"
    assert conn.llen("experience") == 1
    cli.poll()
    assert [cli.take(log("copy"))[:2] for _ in range(2)] == [(0, 1), (1, 2)]
    assert srv.collect_releases(log("wait")) == 2 and srv.free == [0, 1]
    assert wire.wipe_stale_keys(conn) == 3                     # without `keep`: everything, as before
