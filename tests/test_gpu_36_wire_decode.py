"""push_records through the device decode (wire.WireIngest -> b2rl_wire_decode, DESIGN.md §4.24) on one H100: every
store type of the three learners ends up bit for bit where the host decoders put it, also for mixed batches whose
records partly fall back to the host, in list order."""
import ctypes as C
import pickle

import numpy as np
import pytest
import torch

from distributed_rl_b200 import _lib, apex, impala, r2d2
from distributed_rl_b200 import wire as W
from test_wire_template_cpu import _apex, _impala, _r2d2

pytestmark = pytest.mark.gpu
T = 4
CAP = 64


def _host_only(rp):
    rp._wire_decode = lambda blobs: None
    return rp


def _snapshot(rp, sample=True):
    st = rp.store
    n = len(st)
    idx = torch.arange(n, device="cuda")
    snap = {k: v.clone() for k, v in (rp.pool if hasattr(rp, "pool") else st).gather(idx).items()}
    if isinstance(rp, impala.Replay):
        snap["draw"] = rp.draw(min(8, n)).clone()
        return snap
    snap["prio"] = st.priorities(0, n).clone()
    if sample:
        st.seed(11, 0)
        i, _, w = st.sample(8, beta=0.4)
        snap.update(sample_idx=i.clone(), sample_w=w.clone())
    return snap


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k].cpu().view(torch.uint8), b[k].cpu().view(torch.uint8)), k


def _push_both(make, blobs_list):
    dev, host = make(), _host_only(make())
    for blobs in blobs_list:
        dev.push_records(blobs)
        host.push_records(blobs)
    torch.cuda.synchronize()
    assert len(dev.store) == len(host.store) and dev.total_frame == host.total_frame
    return dev, host


APEX_STORES = {"plain": {}, "dedup": dict(FRAME_DEDUP=True), "codec": dict(FRAME_DEDUP=True, FRAME_CODEC=True)}
R2D2_STORES = {"stacks": {}, "strip": dict(FRAME_STRIP=True), "host_frames": dict(FRAME_STRIP=True, HOST_FRAMES=True),
               "dedup": dict(FRAME_DEDUP=True), "host_pool": dict(FRAME_DEDUP=True, HOST_POOL=True),
               "codec": dict(FRAME_DEDUP=True, POOL_CODEC=True)}
IMPALA_STORES = {"plain": {}, "dedup": dict(FRAME_DEDUP=True), "codec": dict(FRAME_DEDUP=True, STAGED_POOL_CODEC=True)}


def _mixed(rng, make_rec, n):
    """Protocol 4 records, with a protocol 2 record (no template: host path) and a protocol 5 one among them."""
    blobs = [pickle.dumps(make_rec(rng, i), protocol=4) for i in range(n)]
    blobs[2] = pickle.dumps(make_rec(rng, 2), protocol=2)
    blobs[5] = pickle.dumps(make_rec(rng, 5), protocol=5)
    return blobs


@pytest.mark.parametrize("store", list(APEX_STORES))
def test_apex_push_records_matches_the_host_decoders(store):
    rng = np.random.default_rng(1)
    make = lambda: apex.Replay(apex.ApexConfig(REPLAY_MEMORY_LEN=CAP, BUFFER_SIZE=0, **APEX_STORES[store]))
    recs = [_apex(rng, i) for i in range(20)]
    recs[6][1] = 300                                    # BININT2: a record of another length, another template
    batches = [[pickle.dumps(r) for r in recs], _mixed(rng, _apex, 12)]
    dev, host = _push_both(make, batches)
    _same(_snapshot(dev), _snapshot(host))
    assert dev._wire.host_records == 1                  # the protocol 2 record only


@pytest.mark.parametrize("store", list(R2D2_STORES))
def test_r2d2_push_records_matches_the_host_decoders(store):
    rng = np.random.default_rng(2)
    cfg = dict(FIXED_TRAJECTORY=T, REPLAY_MEMORY_LEN=CAP, BUFFER_SIZE=0, **R2D2_STORES[store])
    make = lambda: r2d2.Replay(r2d2.R2D2Config(**cfg))
    batches = [[pickle.dumps(_r2d2(rng, i)) for i in range(10)], _mixed(rng, _r2d2, 8)]
    dev, host = _push_both(make, batches)
    _same(_snapshot(dev), _snapshot(host))


@pytest.mark.parametrize("store", list(IMPALA_STORES))
def test_impala_push_records_matches_the_host_decoders(store):
    rng = np.random.default_rng(3)
    make = lambda: impala.Replay(impala.ImpalaConfig(UNROLL_STEP=T, REPLAY_MEMORY_LEN=CAP, BUFFER_SIZE=0,
                                                     **IMPALA_STORES[store]))
    recs = [_impala(rng, i) for i in range(10)]
    recs[4][1] = recs[4][1].copy()
    recs[4][1][1, 0] = 2 ** 33 + 5                      # out of int32: flagged, decoded on the host (astype wraps)
    batches = [[pickle.dumps(r) for r in recs], _mixed(rng, _impala, 8)]
    dev, host = _push_both(make, batches)
    _same(_snapshot(dev), _snapshot(host))
    assert dev._wire.host_records == 2


def test_a_sequence_that_does_not_slide_raises_and_pushes_nothing():
    rng = np.random.default_rng(4)
    rp = r2d2.Replay(r2d2.R2D2Config(FIXED_TRAJECTORY=T, REPLAY_MEMORY_LEN=CAP, BUFFER_SIZE=0, FRAME_STRIP=True))
    rp.push_records([pickle.dumps(_r2d2(rng, i)) for i in range(3)])
    before = len(rp.store)
    blobs = [pickle.dumps(_r2d2(rng, i)) for i in range(5)]
    bad = _r2d2(rng, 3, slide=False)
    blobs[3] = pickle.dumps(bad)
    with pytest.raises(ValueError) as dev_err:
        rp.push_records(blobs)
    with pytest.raises(ValueError) as host_err:
        W.decode_r2d2([pickle.loads(b) for b in blobs], T, strip=True)
    assert str(dev_err.value) == str(host_err.value) and "record 3" in str(dev_err.value)
    assert len(rp.store) == before


def test_wire_decode_rejects_bad_arguments():
    lib = _lib.load()
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    i32 = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = buf.data_ptr()
    fields = (C.c_void_p * 1)(p)
    rows = (C.c_int64 * 1)(16)

    def call(n=1, stride=128, tmpl_len=64, n_runs=1, n_tasks=1, n_fields=1, n_rows=1, blobs=p, f=fields):
        return lib.b2rl_wire_decode(blobs, stride, i32.data_ptr(), n, p, tmpl_len, i32.data_ptr(), n_runs,
                                    i32.data_ptr(), n_tasks, None, f, rows, n_fields, i32.data_ptr(), n_rows, None)
    for bad in (dict(n=-1), dict(stride=64), dict(stride=72), dict(n_runs=0), dict(n_tasks=0), dict(n_tasks=70000),
                dict(n_fields=0), dict(n_fields=9), dict(n_rows=0), dict(blobs=p + 8), dict(f=(C.c_void_p * 1)(None))):
        assert call(**bad) == -1, bad                    # B2RL_ERR_INVALID, before any launch
        assert b"invalid argument" in lib.b2rl_last_error()
    assert call(n=0) == 0
