"""Record templates (wire.derive_template, DESIGN.md §4.24) on the host: a template accounts for every byte of a record
of each kind, and a numpy restatement of b2rl_wire_decode, run from the template, decodes exactly what wire.decode_apex
/ decode_r2d2 / decode_impala decode from the same blobs, or flags the record."""
import pickle

import numpy as np
import pytest
import torch

from distributed_rl_b200 import wire as W

T = 4


def _apex(rng, i):
    s, ns = (rng.integers(0, 256, (4, 84, 84), dtype=np.uint8) for _ in range(2))
    kinds = [(int(rng.integers(6)), float(rng.standard_normal()), bool(i % 2), float(rng.random())),
             (np.int64(rng.integers(6)), np.float64(rng.standard_normal()), np.bool_(i % 2), np.float32(rng.random()))]
    a, r, d, p = kinds[i % 2]
    return [s, a, r, ns, d, p]


def _r2d2(rng, i, numpy_hidden=False, slide=True, T=T):
    frames = rng.integers(0, 256, (T + 3, 84, 84), dtype=np.uint8)
    stacks = [frames[t:t + 4].copy() if slide else rng.integers(0, 256, (4, 84, 84), dtype=np.uint8) for t in range(T)]
    h = [rng.standard_normal((1, 1, 512)).astype(np.float32) for _ in range(2)]
    rec = [tuple(h) if numpy_hidden else tuple(torch.from_numpy(x) for x in h)]
    for t in range(T):
        rec += [stacks[t], int(rng.integers(6)) if t % 2 else np.int64(rng.integers(6)),
                float(rng.standard_normal()) if t % 3 else 0]
    rec.append(bool(i % 2))
    arr = np.empty(len(rec), dtype=object)
    for j, x in enumerate(rec):
        arr[j] = x
    return np.append(arr, float(rng.random()) + 0.1)           # R2D2/Player.py:312-314


def _impala(rng, i, T=T):
    return [rng.integers(0, 256, (T + 1, 28224), dtype=np.uint8), rng.integers(0, 6, (T, 1)),
            rng.uniform(0.05, 0.9, (T, 1)).astype(np.float32 if i % 2 else np.float64), rng.standard_normal(T),
            i % 2]


MAKE = {"apex": _apex, "r2d2": _r2d2, "impala": _impala}


def _host(kind, blobs, strip=False, T=T):
    recs = [pickle.loads(b) for b in blobs]
    if kind == "apex":
        out = {name: np.zeros((len(recs),) + shape, dt) for name, dt, shape in W.record_fields("apex")}
        W.decode_apex(recs, out)
        return out
    cols = W.decode_r2d2(recs, T, strip=strip) if kind == "r2d2" else W.decode_impala(recs, T)
    if kind == "r2d2":
        cols = cols[0] + [cols[1]]
    return {f[0]: c for f, c in zip(W.record_fields(kind, T, strip=strip), cols)}


# ---- the kernel, restated in numpy -----------------------------------------------------------------------------------
_SRC = {W.S_U8: "<u1", W.S_U16: "<u2", W.S_I32: "<i4", W.S_I64: "<i8", W.S_F32: "<f4", W.S_F64: "<f8",
        W.S_F64BE: ">f8"}


def _convert(b: np.ndarray, sk: int, dk: int):
    """One element -> (its bytes in the destination, status bits)."""
    if sk == W.S_BOOLOP:
        if b[0] not in (0x88, 0x89):
            return None, W.STATUS_SKELETON
        v = int(b[0] == 0x88)
    elif sk == W.S_B1:
        v = int(b[0] != 0)
    else:
        v = np.frombuffer(b.tobytes(), _SRC[sk])[0]
    is_float = sk in W.SRC_FLOAT
    truth = bool(v != 0)
    if dk == W.D_I32:
        if is_float:
            return None, W.STATUS_SKELETON
        if not -2 ** 31 <= int(v) < 2 ** 31:
            return None, W.STATUS_RANGE
        return np.int32(int(v)).tobytes(), 0
    if dk in (W.D_F32, W.D_F32_DIRECT):
        if sk == W.S_F32:                       # float() quiets a float32 NaN, numpy's array cast keeps its bits
            bits = int(np.frombuffer(b.tobytes(), "<u4")[0])
            if dk == W.D_F32 and np.isnan(v):
                bits |= 0x400000
            return np.uint32(bits).tobytes(), 0
        if is_float:
            return np.float64(v).astype(np.float32).tobytes(), 0
        if dk == W.D_F32:
            return np.float32(float(int(v))).tobytes(), 0
        return np.int64(v).astype(np.float32).tobytes(), 0
    if dk == W.D_U8_BOOL:
        return bytes([truth]), 0
    return np.float32(0.0 if truth else 1.0).tobytes(), 0


def model_decode(tp: W.Template, blobs):
    n, F = len(blobs), W.FRAME_BYTES
    out = {name: np.zeros((n,) + shape, dt) for name, dt, shape in tp.fields}
    names = [f[0] for f in tp.fields]
    status = np.zeros(n, np.int32)
    ref = np.frombuffer(tp.blob, np.uint8)
    for r, blob in enumerate(blobs):
        b = np.frombuffer(blob, np.uint8)
        if len(b) != tp.length:
            status[r] |= W.STATUS_SKELETON
            continue
        for op, src, ln, f, dst, count, aux, kinds in tp.runs.tolist():
            row = out[names[f]][r:r + 1].reshape(-1).view(np.uint8)
            if op == W.RUN_SKELETON:
                status[r] |= W.STATUS_SKELETON * (not np.array_equal(b[src:src + ln], ref[src:src + ln]))
            elif op == W.RUN_SAME:
                status[r] |= W.STATUS_SKELETON * (not np.array_equal(b[src:src + ln], b[aux:aux + ln]))
            elif op == W.RUN_COPY:
                row[dst:dst + ln] = b[src:src + ln]
            elif op == W.RUN_STRIP:
                if count == 0:
                    row[:4 * F] = b[src:src + 4 * F]
                else:
                    row[(count + 3) * F:(count + 4) * F] = b[src + 3 * F:src + 4 * F]
                if aux >= 0:
                    status[r] |= W.STATUS_NO_SLIDE * (not np.array_equal(b[src + F:src + 4 * F], b[aux:aux + 3 * F]))
            else:
                sk, dk = kinds & 0xFF, kinds >> 8
                sb, db = ln // count, 1 if dk == W.D_U8_BOOL else 4
                for e in range(count):
                    v, st = _convert(b[src + e * sb:src + (e + 1) * sb], sk, dk)
                    status[r] |= st
                    if v is not None:
                        row[dst + e * db:dst + (e + 1) * db] = np.frombuffer(v, np.uint8)
    return out, status


# ---- tests -------------------------------------------------------------------------------------------------------------
def _template(kind, blob, strip=False):
    return W.derive_template(blob, kind, T=T, strip=strip)


@pytest.mark.parametrize("protocol", [3, 4, 5])
@pytest.mark.parametrize("kind", ["apex", "r2d2", "impala"])
def test_a_template_accounts_for_every_byte(kind, protocol):
    rng = np.random.default_rng(protocol)
    blob = pickle.dumps(MAKE[kind](rng, 0), protocol=protocol)
    tp = _template(kind, blob)
    assert tp is not None and tp.length == len(blob)
    cover = np.zeros(len(blob), np.int32)
    for op, src, ln, *_ in tp.runs.tolist():
        cover[src:src + ln] += 1
    for src, ln in tp.free:
        cover[src:src + ln] += 1
    assert (cover >= 1).all()                                            # every byte is in a run or a free span
    skel = np.zeros(len(blob), bool)
    for op, src, ln, *_ in tp.runs.tolist():
        if op == W.RUN_SKELETON:
            skel[src:src + ln] = True
    assert np.array_equal(skel, tp.skeleton) and (cover[skel] == 1).all()   # skeleton overlaps nothing
    values = sum(ln for op, src, ln, *_ in tp.runs.tolist() if op in (W.RUN_COPY, W.RUN_STRIP, W.RUN_CONVERT))
    frames = {"apex": 2 * W.STACK_BYTES, "r2d2": T * W.STACK_BYTES, "impala": (T + 1) * W.STACK_BYTES}[kind]
    assert values > frames                                               # the frames and every scalar are values
    assert int(tp.skeleton.sum()) < 2000 * (T if kind == "r2d2" else 1)
    assert tp.tasks[0, 0] == 0 and tp.tasks[-1, 1] == len(tp.runs) and (tp.tasks[1:, 0] == tp.tasks[:-1, 1]).all()
    if kind == "r2d2":
        assert len(tp.free) == 2                                         # the two torch storage keys


def test_protocol_2_records_take_the_host_path():
    """Protocol 2 pickles bytes as latin-1 text (_codecs.encode), whose length depends on the bytes: no fixed layout."""
    rng = np.random.default_rng(0)
    for kind in MAKE:
        assert _template(kind, pickle.dumps(MAKE[kind](rng, 0), protocol=2)) is None


@pytest.mark.parametrize("kind, strip", [("apex", False), ("r2d2", False), ("r2d2", True), ("impala", False)])
def test_the_kernel_model_equals_the_host_decoders(kind, strip):
    rng = np.random.default_rng(7)
    recs = [MAKE[kind](rng, i) for i in range(6)]
    if kind == "r2d2":
        recs[3] = _r2d2(rng, 3, numpy_hidden=True)
    blobs = [pickle.dumps(r, protocol=4) for r in recs]
    by_len = {}
    for i, b in enumerate(blobs):
        by_len.setdefault(len(b), []).append(i)
    want = _host(kind, blobs, strip)
    for pos in by_len.values():
        tp = _template(kind, blobs[pos[0]], strip)
        assert tp is not None
        got, status = model_decode(tp, [blobs[i] for i in pos])
        assert (status == 0).all()
        for name in want:
            assert got[name].dtype == want[name].dtype
            np.testing.assert_array_equal(got[name].view(np.uint8), want[name][pos].view(np.uint8), err_msg=name)


SNAN32 = np.array([0x7F800001, 0xFFA00000], np.uint32).view(np.float32)     # signalling NaNs, low / high payload


def test_float32_nans_decode_like_the_host():
    """Signalling float32 NaNs in scalar fields (float(x): quieted) and in arrays and LSTM states (the array cast: bits
    kept), through the templates derive_template builds."""
    rng = np.random.default_rng(8)
    apex = _apex(rng, 1)
    apex[2], apex[5] = SNAN32[0], SNAN32[1]
    r2d2 = _r2d2(rng, 0)
    h = rng.standard_normal((2, 1, 1, 512)).astype(np.float32)
    h[:, 0, 0, 5:7] = SNAN32
    r2d2[0] = (torch.from_numpy(h[0]), h[1])
    r2d2[3], r2d2[-1] = SNAN32[1], SNAN32[0]
    imp = _impala(rng, 1)
    imp[2][1:3, 0] = SNAN32
    imp[3] = imp[3].astype(np.float32)
    imp[3][0], imp[4] = SNAN32[0], SNAN32[1]
    for kind, rec in (("apex", apex), ("r2d2", r2d2), ("impala", imp)):
        blob = pickle.dumps(rec, protocol=4)
        got, status = model_decode(_template(kind, blob), [blob])
        want = _host(kind, [blob])
        assert status.tolist() == [0]
        for name in want:
            np.testing.assert_array_equal(got[name].view(np.uint8), want[name].view(np.uint8), err_msg=f"{kind} {name}")


def test_float_conversions_round_like_numpy():
    """fp64 -> fp32 rounds to nearest even, overflows to inf and keeps a NaN's payload top, as the host cast does; a
    float32 scalar's signalling NaN is quieted, as float() quiets it, while a float32 array element keeps its bits."""
    for bits in (0x7F800001, 0xFF800001, 0x7FA00000, 0xFFBFFFFF, 0x7FC00001, 0x00000001, 0x7F7FFFFF, 0xFF800000):
        x = np.array([bits], np.uint32).view(np.float32)
        src = np.frombuffer(x.tobytes(), np.uint8)
        host = np.zeros(1, np.float32)
        host[0] = float(x[0])                                       # decode_apex / decode_r2d2 / decode_impala scalars
        assert _convert(src, W.S_F32, W.D_F32)[0] == host.tobytes(), hex(bits)
        assert _convert(src, W.S_F32, W.D_F32_DIRECT)[0] == np.asarray(x, np.float32).tobytes(), hex(bits)
    vals = np.array([1 + 2 ** -24, 1 + 3 * 2 ** -24, 3.4e38, 1e300, -1e-50, np.nan, -np.inf, 16777217.0])
    vals = np.concatenate([vals, np.frombuffer(np.array([0x7FF0000000000123, 0xFFF8000012345678], np.uint64), np.float64)])
    for v in vals:
        got, _ = _convert(np.frombuffer(np.float64(v).tobytes()[::-1], np.uint8), W.S_F64BE, W.D_F32)
        host = np.zeros(1, np.float32)
        host[0] = float(v)
        assert got == host.tobytes(), v
    for i in (2 ** 24 + 1, 2 ** 53 + 1, -(2 ** 62) - 1):
        host = np.zeros(1, np.float32)
        host[0] = float(i)
        assert _convert(np.frombuffer(np.int64(i).tobytes(), np.uint8), W.S_I64, W.D_F32)[0] == host.tobytes()
        assert _convert(np.frombuffer(np.int64(i).tobytes(), np.uint8), W.S_I64, W.D_F32_DIRECT)[0] == \
            np.array([i], np.int64).astype(np.float32).tobytes()


def _flag(kind, blob, mutate):
    tp = _template(kind, blob)
    bad = mutate(bytearray(blob), tp)
    return model_decode(tp, [bytes(bad)])[1][0]


def _run_of(tp, field, op=W.RUN_CONVERT):
    names = [f[0] for f in tp.fields]
    return next(r for r in tp.runs.tolist() if r[0] == op and r[3] == names.index(field))


def test_a_changed_scalar_opcode_is_a_skeleton_mismatch():
    blob = pickle.dumps([np.zeros((4, 84, 84), np.uint8), 3, 0.5, np.zeros((4, 84, 84), np.uint8), True, 1.0])

    def swap(b, tp):
        at = _run_of(tp, "r")[1] - 1            # BINFLOAT 'G' -> another opcode, same length
        assert b[at] == ord("G")
        b[at] = ord("J")
        return b
    assert _flag("apex", blob, swap) == W.STATUS_SKELETON

    def flip(b, tp):                             # NEWTRUE -> NONE: a value span that is not a bool opcode
        at = _run_of(tp, "d")[1]
        b[at] = ord("N")
        return b
    assert _flag("apex", blob, flip) & W.STATUS_SKELETON


def test_a_changed_length_and_a_truncated_blob_are_skeleton_mismatches():
    rng = np.random.default_rng(3)
    blob = pickle.dumps(_impala(rng, 0), protocol=4)

    def length(b, tp):
        at = _run_of(tp, "state", W.RUN_COPY)[1] - 8       # the BINBYTES8 length in front of the frames
        b[at] ^= 1
        return b
    assert _flag("impala", blob, length) == W.STATUS_SKELETON
    assert _flag("impala", blob, lambda b, tp: b[:-1]) == W.STATUS_SKELETON


def test_an_out_of_range_action_is_flagged_not_wrapped():
    rng = np.random.default_rng(4)
    rec = _apex(rng, 1)
    blob = pickle.dumps(rec)
    tp = _template("apex", blob)
    rec[1] = np.int64(2 ** 40)
    out, status = model_decode(tp, [pickle.dumps(rec)])
    assert status[0] == W.STATUS_RANGE
    imp = _impala(rng, 0)
    tp = _template("impala", pickle.dumps(imp))
    imp[1] = imp[1].copy()
    imp[1][2, 0] = -(2 ** 31) - 1
    assert model_decode(tp, [pickle.dumps(imp)])[1][0] == W.STATUS_RANGE


def test_a_sequence_that_does_not_slide_is_flagged():
    rng = np.random.default_rng(5)
    good = pickle.dumps(_r2d2(rng, 0, numpy_hidden=True))       # numpy LSTM states: no storage key, one length
    tp = _template("r2d2", good, strip=True)
    bad = pickle.dumps(_r2d2(rng, 0, numpy_hidden=True, slide=False))
    assert len(bad) == len(good)
    assert model_decode(tp, [good, bad])[1].tolist() == [0, W.STATUS_NO_SLIDE]
