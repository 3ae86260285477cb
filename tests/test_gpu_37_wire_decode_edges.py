"""b2rl_wire_decode (csrc/wire.cu, DESIGN.md §4.24) launched directly on one H100 against the host decoders
(wire.decode_apex / decode_r2d2 / decode_impala), bit for bit: records at the learners' lengths (R2D2 at T = 80, IMPALA
at T = 20), every conversion edge in every value slot a template produces, and records corrupted one at a time.  Every
record's status word is read: a record with status 0 must equal the host decoders in every field, a flagged record must
carry exactly the status the test predicts, which the numpy restatement of the kernel (model_decode) predicts too."""
import ctypes as C
import pickle
import struct

import numpy as np
import pytest
import torch

from distributed_rl_b200 import _lib, apex, impala, r2d2
from distributed_rl_b200 import wire as W
from test_gpu_36_wire_decode import _push_both, _same, _snapshot
from test_wire_template_cpu import _apex, _host, _impala, _r2d2, model_decode

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5                  # what the field rows hold before the launch
T_R2D2, T_IMPALA = 80, 20        # the learners' sequence and rollout lengths
F = W.FRAME_BYTES


# ---- the launch ------------------------------------------------------------------------------------------------------
def _min_stride(length):
    return (length + 16 + 15) // 16 * 16


def _decode(tp, blobs, rows=None, n_rows=None, stride=None):
    """b2rl_wire_decode of `blobs` against `tp`, staged as WireIngest.decode stages them: record i at i * stride (the
    smallest multiple of 16 with 16 bytes to spare unless given), junk between the blobs, the device buffer ending at
    the last record's stride.  rows: the row of each record (an int32 permutation into n_rows), or None for row i.
    -> ({field: (n_rows, *shape) numpy array}, status (n_rows,) int32)"""
    n = len(blobs)
    n_rows = n if n_rows is None else n_rows
    stride = stride or _min_stride(tp.length)
    stage = np.full(n * stride, 0xEE, np.uint8)
    for i, b in enumerate(blobs):
        stage[i * stride:i * stride + len(b)] = np.frombuffer(b, np.uint8)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    staged, lengths = dev(stage), dev(np.array([len(b) for b in blobs], np.int32))
    tmpl, runs, tasks = dev(np.frombuffer(tp.blob, np.uint8)), dev(tp.runs), dev(tp.tasks)
    rows_dev = None if rows is None else dev(np.asarray(rows, np.int32))
    fields = [torch.full((n_rows, int(np.prod(shape, dtype=np.int64)) * np.dtype(dt).itemsize), SENTINEL,
                         dtype=torch.uint8, device="cuda") for _, dt, shape in tp.fields]
    status = torch.zeros(n_rows, dtype=torch.int32, device="cuda")
    lib = _lib.load()
    rc = lib.b2rl_wire_decode(staged.data_ptr(), stride, lengths.data_ptr(), n, tmpl.data_ptr(), tp.length,
                              runs.data_ptr(), len(tp.runs), tasks.data_ptr(), len(tp.tasks),
                              None if rows_dev is None else rows_dev.data_ptr(),
                              (C.c_void_p * len(fields))(*[f.data_ptr() for f in fields]),
                              (C.c_int64 * len(fields))(*[f.shape[1] for f in fields]), len(fields),
                              status.data_ptr(), n_rows, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.b2rl_last_error()
    torch.cuda.synchronize()
    out = {name: f.cpu().numpy().view(dt).reshape((n_rows,) + shape) for f, (name, dt, shape) in zip(fields, tp.fields)}
    return out, status.cpu().numpy()


def _equal_bits(got, want, what):
    g, w = got.reshape(len(got), -1), want.reshape(len(want), -1)
    bad = np.flatnonzero((g.view(np.uint8).reshape(len(g), -1) != w.view(np.uint8).reshape(len(w), -1)).any(1))
    if len(bad):
        r = bad[0]
        k = np.flatnonzero(g[r].view(np.uint8) != w[r].view(np.uint8))[0] // g.itemsize
        word = lambda x: x[r].view(f"u{g.itemsize}")[k]
        raise AssertionError(f"{what}: records {bad.tolist()[:8]} differ, first at record {r} element {k}: "
                             f"{word(g):#x} decoded, {word(w):#x} from the host")


def _check(tp, blobs, expect, got, status, rows=None, T=0, strip=False):
    """Each record's status is expect[i], as model_decode predicts; a record with status 0 equals the host decoders in
    every field, bit for bit; a record of another length than the template's leaves its row at the sentinel; rows that
    no record names keep the sentinel and status 0."""
    n = len(blobs)
    rows = np.arange(n) if rows is None else np.asarray(rows)
    expect = np.asarray(expect, np.int32)
    with np.errstate(all="ignore"):                 # float32 overflow in the host casts is part of what is compared
        assert model_decode(tp, blobs)[1].tolist() == expect.tolist()
        assert status[rows].tolist() == expect.tolist()
        ok = np.flatnonzero(expect == 0)
        want = _host(tp.kind, [blobs[i] for i in ok], strip, T) if len(ok) else {}
        for name in want:
            _equal_bits(got[name][rows[ok]], want[name], f"{tp.kind} {name}")
    unnamed = np.setdiff1d(np.arange(len(status)), rows)
    assert (status[unnamed] == 0).all()
    untouched = np.concatenate([rows[[len(b) != tp.length for b in blobs]], unnamed])
    for name in got:
        assert (got[name][untouched].view(np.uint8) == SENTINEL).all(), name


def _by_layout(blobs, kind, T=0, strip=False):
    """{template digest: (Template, indices of the blobs of that layout)}, each template derived from its first blob."""
    groups = {}
    for i, b in enumerate(blobs):
        tp = W.derive_template(b, kind, T=T, strip=strip)
        assert tp is not None, i
        groups.setdefault(tp.digest, (tp, []))[1].append(i)
    return groups


def _decode_and_check(kind, blobs, expect, T=0, strip=False, spare_rows=3, seed=0):
    """Every layout among `blobs` launched once, its records scattered to a random permutation of spare_rows more
    rows than it has, and checked.  -> the templates"""
    rng = np.random.default_rng(seed)
    tps = []
    for tp, pos in _by_layout(blobs, kind, T, strip).values():
        n_rows = len(pos) + spare_rows
        rows = rng.permutation(n_rows)[:len(pos)]
        sub = [blobs[i] for i in pos]
        got, status = _decode(tp, sub, rows, n_rows)
        _check(tp, sub, [expect[i] for i in pos], got, status, rows, T, strip)
        tps.append(tp)
    return tps


# ---- records at the learners' lengths -----------------------------------------------------------------------------
def _records(kind, n, seed=0):
    """Protocol 4 pickles as the reference Players make them (torch LSTM states), with Python and numpy scalars mixed as
    test_wire_template_cpu's record makers mix them."""
    rng = np.random.default_rng(seed)
    if kind == "apex":
        return [pickle.dumps(_apex(rng, i), protocol=4) for i in range(n)]
    if kind == "r2d2":
        return [pickle.dumps(_r2d2(rng, i, T=T_R2D2), protocol=4) for i in range(n)]
    return [pickle.dumps(_impala(rng, i, T=T_IMPALA), protocol=4) for i in range(n)]


BATCHES = {"apex": (1024, 0, False), "r2d2_strips": (32, T_R2D2, True), "r2d2_stacks": (32, T_R2D2, False),
           "impala": (128, T_IMPALA, False)}        # tools/bench_wire_ingest.py's batches


@pytest.fixture(scope="module")
def batches():
    return {kind: _records(kind, BATCHES[f"{kind}_strips" if kind == "r2d2" else kind][0])
            for kind in ("apex", "r2d2", "impala")}


@pytest.mark.parametrize("batch", list(BATCHES))
def test_records_at_the_learners_lengths_decode_like_the_host(batches, batch):
    n, T, strip = BATCHES[batch]
    kind = batch.split("_")[0]
    tps = _decode_and_check(kind, batches[kind], [0] * n, T, strip)
    if kind == "r2d2":
        for tp in tps:
            frames = [r for r in tp.runs.tolist() if r[0] in (W.RUN_COPY, W.RUN_STRIP)]
            assert len(frames) == T
            # every source phase mod 16, so every shift16 branch copies frames (a strip's later stacks copy from
            # src + 3 frames, and 3 * 7056 is a multiple of 16)
            assert {r[1] % 16 for r in frames} == set(range(16))
            assert len(tp.tasks) == 41


PUSH_STORES = {
    "apex": {"dedup": dict(FRAME_DEDUP=True), "codec": dict(FRAME_DEDUP=True, FRAME_CODEC=True)},
    "r2d2": {"dedup": dict(FRAME_DEDUP=True), "codec": dict(FRAME_DEDUP=True, POOL_CODEC=True)},
    "impala": {"dedup": dict(FRAME_DEDUP=True), "codec": dict(FRAME_DEDUP=True, STAGED_POOL_CODEC=True)},
}


@pytest.mark.parametrize("store", ["dedup", "codec"])
@pytest.mark.parametrize("kind", ["apex", "r2d2", "impala"])
def test_push_records_at_the_learners_lengths_decodes_every_record_on_the_device(batches, kind, store):
    blobs = batches[kind]
    kw = PUSH_STORES[kind][store]
    if kind == "apex":
        make = lambda: apex.Replay(apex.ApexConfig(REPLAY_MEMORY_LEN=len(blobs), BUFFER_SIZE=0, **kw))
    elif kind == "r2d2":
        make = lambda: r2d2.Replay(r2d2.R2D2Config(FIXED_TRAJECTORY=T_R2D2, REPLAY_MEMORY_LEN=len(blobs),
                                                   BUFFER_SIZE=0, **kw))
    else:
        make = lambda: impala.Replay(impala.ImpalaConfig(UNROLL_STEP=T_IMPALA, REPLAY_MEMORY_LEN=len(blobs),
                                                         BUFFER_SIZE=0, **kw))
    dev, host = _push_both(make, [blobs])
    assert dev._wire.host_records == 0
    _same(_snapshot(dev), _snapshot(host))


# ---- conversion edges ------------------------------------------------------------------------------------------------
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
WIDE = 2 ** 60 + 2 ** 36 + 1     # float() then float32 rounds it to 0x5d800000, numpy's int64 -> float32 to 0x5d800001
TIE = (2 - 2 ** -24) * 2.0 ** 127                    # rounds to inf in float32


def _f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


F32_BITS = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x3F800001, 0x7F7FFFFF, 0xFF7FFFFF,
            0x7F800000, 0xFF800000,
            0x7FE00000, 0xFFE00000, 0x7FC00001, 0xFFC00001,      # quiet NaNs: payload in the high / the low bits
            0x7FA00000, 0xFFA00000, 0x7F800001, 0xFF800001]      # signalling NaNs
F64_VALUES = [0.0, -0.0, 2.0 ** -149, -2.0 ** -149, (2 ** 23 - 1) * 2.0 ** -149, _f64(1), -_f64(1),
              _f64(0x000FFFFFFFFFFFFF), 2.0 ** -150, -2.0 ** -150, 3 * 2.0 ** -151, 1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24,
              float(np.finfo(np.float32).max), TIE, float(np.nextafter(TIE, 0.0)), -TIE, float("inf"), float("-inf")]
F64_VALUES += [_f64(b) for b in (0x7FFC000000000000, 0xFFFC000000000000, 0x7FF8000000000001, 0xFFF8000000000001,
                                 0x7FF4000000000000, 0xFFF4000000000000, 0x7FF0000000000001, 0xFFF0000000000001)]
F32_VALUES = list(np.array(F32_BITS, np.uint32).view(np.float32))
# integers by numpy dtype; the out-of-int32 ones are flagged ST_RANGE in D_I32 fields and converted in float ones
INTS = {"<i8": [0, -1, I32_MIN, I32_MAX, 2 ** 24 + 1], "<i4": [0, -1, I32_MIN, I32_MAX, 2 ** 24 + 1],
        "|u1": [0, 1, 255], "<u2": [0, 256, 65535]}
WIDE_INTS = [I32_MIN - 1, I32_MAX + 1, WIDE, -WIDE, 2 ** 53 + 1, -2 ** 63, 2 ** 63 - 1]
PY_INTS = [0, 1, 255, 256, 65535, 65536, -1, I32_MIN, I32_MAX]            # BININT1, BININT2, BININT
INT_SCALARS = (PY_INTS + [True, False] + [np.int64(v) for v in INTS["<i8"]] + [np.int32(v) for v in INTS["<i4"]]
               + [np.uint8(v) for v in INTS["|u1"]] + [np.uint16(v) for v in INTS["<u2"]]
               + [np.bool_(True), np.bool_(False)])
SCALARS = (INT_SCALARS + [np.int64(v) for v in WIDE_INTS] + F64_VALUES + [np.float64(v) for v in F64_VALUES]
           + F32_VALUES)
ARRAYS = {"<f8": np.array(F64_VALUES), "<f4": np.array(F32_BITS, np.uint32).view(np.float32),
          "<i8": np.array(INTS["<i8"] + WIDE_INTS),
          "<i4": np.array(INTS["<i4"], np.int32), "|u1": np.array(INTS["|u1"], np.uint8),
          "<u2": np.array(INTS["<u2"], np.uint16), "|b1": np.array([True, False, True])}
INT_ARRAYS = {"<i8": np.array(INTS["<i8"], np.int64), "<i4": ARRAYS["<i4"], "|u1": ARRAYS["|u1"], "<u2": ARRAYS["<u2"]}


def _array(values, j, n, dt):
    return np.resize(np.roll(values, -j), n).astype(dt)


def _covered(tps, want):
    """The (field, source kind, destination kind) of every converting run of `tps` include `want`."""
    seen = set()
    for tp in tps:
        names = [f[0] for f in tp.fields]
        seen |= {(names[r[3]], r[7] & 0xFF, r[7] >> 8) for r in tp.runs.tolist() if r[0] == W.RUN_CONVERT}
    assert want <= seen, sorted(want - seen)


ALL_SRC = set(range(len(W.SRC_BYTES)))
INT_SRC = ALL_SRC - set(W.SRC_FLOAT)
ARRAY_SRC = {W.S_F64, W.S_F32, W.S_I64, W.S_I32, W.S_U8, W.S_U16, W.S_B1}


def test_conversion_edges_in_apex_scalars():
    """a: every integer kind (D_I32); r, p: every scalar kind (float(x), D_F32); d: every scalar kind (bool(x))."""
    rng = np.random.default_rng(10)
    s, ns = rng.integers(0, 256, (2, 4, 84, 84), dtype=np.uint8)
    n = len(SCALARS)
    recs = [[s, INT_SCALARS[j % len(INT_SCALARS)], SCALARS[j], ns, SCALARS[(j + 7) % n], SCALARS[(j + 13) % n]]
            for j in range(n)]
    recs += [[s, np.int64(v), 0.5, ns, False, 1.0] for v in WIDE_INTS]
    expect = [0] * n + [W.STATUS_RANGE] * len(WIDE_INTS)
    tps = _decode_and_check("apex", [pickle.dumps(r, protocol=4) for r in recs], expect)
    _covered(tps, {("a", k, W.D_I32) for k in INT_SRC} | {(f, k, W.D_F32) for f in "rp" for k in ALL_SRC}
             | {("d", k, W.D_U8_BOOL) for k in ALL_SRC})


def test_conversion_edges_in_r2d2_scalars_and_lstm_states():
    """action: integer kinds; reward, p: every scalar kind (D_F32); done: every scalar kind (notdone = float(not x));
    h0 / h1: torch float32 storages and numpy arrays of every dtype (the array cast, D_F32_DIRECT)."""
    T, hidden = 4, 512
    rng = np.random.default_rng(11)
    frames = rng.integers(0, 256, (T + 3, 84, 84), dtype=np.uint8)
    n, ni = len(SCALARS), len(INT_SCALARS)
    states = ["torch"] + list(ARRAYS)

    def state(k, j):
        x = _array(ARRAYS[k] if k != "torch" else ARRAYS["<f4"], j, hidden, k if k != "torch" else "<f4")
        x = x.reshape(1, 1, hidden)
        return torch.from_numpy(x) if k == "torch" else x

    def record(j, action=None):
        rec = np.empty(3 * T + 3, object)
        rec[0] = (state(states[j % len(states)], j), state(states[(j + 3) % len(states)], j + 1))
        for t in range(T):
            rec[1 + 3 * t] = frames[t:t + 4].copy()
            rec[2 + 3 * t] = INT_SCALARS[(j * T + t) % ni] if action is None else (action if t == 2 else 1)
            rec[3 + 3 * t] = SCALARS[(j * T + t + 5) % n]
        rec[-2], rec[-1] = SCALARS[j], SCALARS[(j + 11) % n]
        return rec

    recs = [record(j) for j in range(n)] + [record(j, np.int64(v)) for j, v in enumerate(WIDE_INTS)]
    expect = [0] * n + [W.STATUS_RANGE] * len(WIDE_INTS)
    tps = _decode_and_check("r2d2", [pickle.dumps(r, protocol=4) for r in recs], expect, T, strip=True)
    _covered(tps, {("action", k, W.D_I32) for k in INT_SRC}
             | {(f, k, W.D_F32) for f in ("reward", "p") for k in ALL_SRC}
             | {("notdone", k, W.D_F32_NOT) for k in ALL_SRC}
             | {(f, k, W.D_F32_DIRECT) for f in ("h0", "h1") for k in ARRAY_SRC})


def test_conversion_edges_in_impala_arrays_and_done():
    """action: arrays of every integer dtype (D_I32); mu, reward: arrays of every dtype (the array cast,
    D_F32_DIRECT); done: every scalar kind (D_F32)."""
    T = T_IMPALA
    rng = np.random.default_rng(12)
    state = rng.integers(0, 256, (T + 1, W.STACK_BYTES), dtype=np.uint8)
    n = len(SCALARS)
    ints, dts = list(INT_ARRAYS), list(ARRAYS)
    recs = [[state, _array(INT_ARRAYS[ints[j % 4]], j, T, ints[j % 4]).reshape(T, 1),
             _array(ARRAYS[dts[j % 7]], j, T, dts[j % 7]).reshape(T, 1), _array(ARRAYS[dts[(j + 3) % 7]], j, T,
                                                                                  dts[(j + 3) % 7]), SCALARS[j]]
            for j in range(n)]
    for j, v in enumerate(WIDE_INTS):
        a = np.ones((T, 1), np.int64)
        a[j % T] = v
        recs.append([state, a, np.full((T, 1), 0.5, np.float32), np.zeros(T), 1])
    expect = [0] * n + [W.STATUS_RANGE] * len(WIDE_INTS)
    tps = _decode_and_check("impala", [pickle.dumps(r, protocol=4) for r in recs], expect, T)
    _covered(tps, {("action", k, W.D_I32) for k in (W.S_I64, W.S_I32, W.S_U8, W.S_U16)}
             | {(f, k, W.D_F32_DIRECT) for f in ("mu", "reward") for k in ARRAY_SRC}
             | {("done", k, W.D_F32) for k in ALL_SRC})


# ---- corrupted records -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def clean():
    """Per kind: the template and three clean records of its length (R2D2: T = 80 strips with torch LSTM states,
    IMPALA: T = 20 with float32 mu)."""
    out = {}
    for kind, T, strip, make in (("r2d2", T_R2D2, True, lambda rng, i: _r2d2(rng, i, T=T_R2D2)),
                                 ("impala", T_IMPALA, False, lambda rng, i: _impala(rng, 1, T=T_IMPALA))):
        rng = np.random.default_rng(13)
        blobs = [pickle.dumps(make(rng, i), protocol=4) for i in range(6)]
        blobs = [b for b in blobs if len(b) == len(blobs[0])][:3]
        assert len(blobs) == 3
        out[kind] = (W.derive_template(blobs[0], kind, T=T, strip=strip), blobs, T, strip)
    assert len(out["r2d2"][0].tasks) == 41 and len(out["impala"][0].tasks) == 2
    return out


def _skeleton_byte(tp, task):
    """A byte in the middle of the longest skeleton run of CTA `task`."""
    lo, hi = tp.tasks[task]
    skel = [r for r in tp.runs[lo:hi].tolist() if r[0] == W.RUN_SKELETON]
    assert skel, task
    r = max(skel, key=lambda r: r[2])
    return r[1] + r[2] // 2


def _strip_run(tp, t):
    return next(r for r in tp.runs.tolist() if r[0] == W.RUN_STRIP and r[5] == t)


def _flip(b, at):
    b[at] ^= 0x5A


def _break_slide(b, tp, t, last):
    """Stacks t and t + 1 no longer overlap: the first byte of the overlap changed in stack t + 1, or its last byte in
    stack t (each copy is read by this pair's check alone)."""
    src, aux = _strip_run(tp, t)[1], _strip_run(tp, t)[6]
    _flip(b, src + 4 * F - 1 if last else aux)


def _storage_key(b, tp, both):
    """h0's torch storage key changed to another digit string of its length, where it first appears and, with `both`,
    where the key list repeats it."""
    same = next(r for r in tp.runs.tolist() if r[0] == W.RUN_SAME)
    key_at, again_at, n = same[6], same[1], same[2]
    new = bytes((c - 48 + 1) % 10 + 48 for c in b[key_at:key_at + n])
    b[key_at:key_at + n] = new
    if both:
        b[again_at:again_at + n] = new


def _cases(kind, tp):
    K = len(tp.tasks)
    ST_S, ST_N = W.STATUS_SKELETON, W.STATUS_NO_SLIDE
    cases = {f"skeleton_task_{k}": (lambda b, k=k: _flip(b, _skeleton_byte(tp, k)), ST_S) for k in (0, K // 2, K - 1)}
    if kind == "r2d2":
        cases["key_in_both_places"] = (lambda b: _storage_key(b, tp, True), 0)
        cases["key_in_one_place"] = (lambda b: _storage_key(b, tp, False), ST_S)
        for t in (0, 39, 78):
            for last in (False, True):
                cases[f"slide_{t}_{t + 1}_{'last' if last else 'first'}"] = (
                    lambda b, t=t, last=last: _break_slide(b, tp, t, last), ST_N)
        cases["skeleton_and_slide"] = (lambda b: (_flip(b, _skeleton_byte(tp, 0)), _break_slide(b, tp, 39, True)),
                                       ST_S | ST_N)
    return cases


CASES = {"r2d2": ["skeleton_task_0", "skeleton_task_mid", "skeleton_task_last", "short", "long", "key_in_both_places",
                  "key_in_one_place", "slide_0_1_first", "slide_0_1_last", "slide_39_40_first", "slide_39_40_last",
                  "slide_78_79_first", "slide_78_79_last", "skeleton_and_slide"],
         "impala": ["skeleton_task_0", "skeleton_task_last", "short", "long"]}      # an IMPALA record is two CTAs


@pytest.mark.parametrize("kind, case", [(k, c) for k, cases in CASES.items() for c in cases])
def test_a_corrupted_record_is_flagged_and_its_neighbours_decode(clean, kind, case):
    tp, blobs, T, strip = clean[kind]
    K = len(tp.tasks)
    bad = bytearray(blobs[1])
    if case == "short":
        bad, want = bad[:-1], W.STATUS_SKELETON
    elif case == "long":
        bad, want = bad + b"\x00", W.STATUS_SKELETON
    else:
        name = case.replace("task_mid", f"task_{K // 2}").replace("task_last", f"task_{K - 1}")
        mutate, want = _cases(kind, tp)[name]
        mutate(bad)
    batch = [blobs[0], bytes(bad), blobs[2]]
    rows = np.array([3, 0, 2])
    results = []
    for stride in (_min_stride(tp.length), _min_stride(tp.length) + 48):
        got, status = _decode(tp, batch, rows, 5, stride)
        _check(tp, batch, [0, want, 0], got, status, rows, T, strip)
        results.append((got, status))
    (g0, s0), (g1, s1) = results
    assert np.array_equal(s0, s1) and all(np.array_equal(g0[k].view(np.uint8), g1[k].view(np.uint8)) for k in g0)
