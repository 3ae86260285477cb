"""The Redis-facing edge of the three learners: what crosses the actor <-> learner wire and how it
is decoded into the HBM replay's fixed field layouts.

The wire itself (Redis lists / keys of pickled blobs, SURVEY.md §5) is the reference's and is out of
scope; this module only keeps UNMODIFIED actors working against the device-resident learners:

  list  "experience"   Ape-X  [s, a, R_n, s', done, prio]                 APE_X/Player.py:252-261
                       R2D2   [(h0,h1), (s,a,r) x T, done, prio]          R2D2/Player.py:38-63,312-319
  list  "trajectory"   IMPALA [s[T+1,28224], a[T,1], mu[T,1], r[T], flag] IMPALA/Player.py:97-114,183-190
  list  "reward"       episode returns, drained every 500 learner steps   APE_X/Learner.py:219-230
  keys  state_dict / target_state_dict / count / Start                    APE_X/Learner.py:149-155,207-216
        params / Count                                                    IMPALA/Learner.py:286-287

`connect` is anything with redis-py's StrictRedis surface (pipeline / lrange / delete / set / get / scan).
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import torch


def drain(connect, key: str) -> list:
    """Atomically take everything queued under list `key`.

    The reference reads with LRANGE 0 -1 + LTRIM -1 0 inside one MULTI and then DELETEs the key outside
    of it (APE_X/ReplayMemory.py:128-133).  LTRIM -1 0 keeps a ONE-element list intact (start = stop = 0),
    so without the DELETE a lone record is re-read on every poll; with the DELETE outside the transaction,
    records pushed between EXEC and DELETE are lost.  LRANGE + DELETE inside the same MULTI has neither
    problem and is what this does."""
    pipe = connect.pipeline()
    pipe.lrange(key, 0, -1)
    pipe.delete(key)
    return list(pipe.execute()[0] or [])


def wipe_stale_keys(connect, keep=()) -> int:
    """Learner.__init__ (APE_X/Learner.py:41-43, R2D2/Learner.py:54,63-64): drop whatever a previous run
    left in the database (stale `experience`, `Start`, parameters ...).  `keep`: key names that belong to a
    process which is already running beside the learner (a replay server) and are left alone."""
    names = connect.scan()
    keys = list(names[-1]) if names else []
    if keep:
        keep = set(keep)
        keys = [k for k in keys if (k.decode() if isinstance(k, bytes) else k) not in keep]
    if keys:
        connect.delete(*keys)
    return len(keys)


def drain_rewards(connect, default: float = -21.0):
    """Every 500 steps the reference averages and clears the actors' `reward` list
    (APE_X/Learner.py:219-230; -21 when nothing arrived).  -> (mean reward, n)"""
    data = drain(connect, "reward")
    if not data:
        return default, 0
    return float(sum(float(pickle.loads(d)) for d in data) / len(data)), len(data)


def checkpoint_path(log_w: str | None) -> str | None:
    """./weight/<ALG>/<time>/weight.pth (APE_X/Learner.py:256-262); the directory is made on first use."""
    if not log_w:
        return None
    os.makedirs(log_w, exist_ok=True)
    return os.path.join(log_w, "weight.pth")


# ---------------------------------------------------------------------------------------------
# record decoders: pickled actor records -> per-field arrays in the replay's layout
# ---------------------------------------------------------------------------------------------
def decode_apex(recs, out) -> None:
    """recs: unpickled [s, a, R_n, s', done, prio]; out: dict of numpy views s/ns/a/r/d/p (len >= n)."""
    s, ns, a, rw, d, p = (out[k] for k in ("s", "ns", "a", "r", "d", "p"))
    for i, r in enumerate(recs):
        s[i] = np.asarray(r[0], np.uint8).reshape(s.shape[1:])
        ns[i] = np.asarray(r[3], np.uint8).reshape(ns.shape[1:])
        a[i], rw[i], d[i], p[i] = int(r[1]), float(r[2]), bool(r[4]), float(r[5])


def _hidden(h, hidden: int) -> np.ndarray:
    t = h.detach().cpu().numpy() if torch.is_tensor(h) else np.asarray(h)
    return t.reshape(-1)[:hidden].astype(np.float32)


def decode_r2d2(recs, T: int, hidden: int = 512, strip: bool = False):
    """R2D2 records (object arrays): rec[0] = (h0, h1) each (1,1,hidden); rec[1+3t], rec[2+3t], rec[3+3t]
    = s_t (4,84,84) u8, a_t, r_t; rec[-2] = done; rec[-1] = priority.  Exactly the indexing of
    R2D2/ReplayMemory.py:70-88 (`done` becomes notdone = float(not done), :86).
    `strip`: state is written as frame strips (n, T + 3, 84, 84) straight from the records (replay.encode_strip); a
    record whose stacks do not slide raises ValueError naming its position, before anything is returned.
    -> ([state, action, reward, h0, h1, notdone], priorities)"""
    from .replay import encode_strip
    n = len(recs)
    s = np.empty((n, T + 3, 84, 84) if strip else (n, T, 4, 84, 84), np.uint8)
    a = np.empty((n, T), np.int32)
    rw = np.empty((n, T), np.float32)
    h0 = np.empty((n, hidden), np.float32)
    h1 = np.empty((n, hidden), np.float32)
    nd = np.empty(n, np.float32)
    p = np.empty(n, np.float32)
    for i, r in enumerate(recs):
        h0[i], h1[i] = _hidden(r[0][0], hidden), _hidden(r[0][1], hidden)
        if strip:
            encode_strip((r[1 + 3 * t] for t in range(T)), s[i], i)
        for t in range(T):
            if not strip:
                s[i, t] = np.asarray(r[1 + 3 * t], np.uint8).reshape(4, 84, 84)
            a[i, t] = int(r[2 + 3 * t])
            rw[i, t] = float(r[3 + 3 * t])
        nd[i] = float(not r[-2])
        p[i] = float(r[-1])
    return [s, a, rw, h0, h1, nd], p


def decode_impala(recs, T: int):
    """IMPALA rollouts: [s (T+1, 28224) u8, a (T,1), mu (T,1), r (T,), flag] with flag = 0 at episode end
    (IMPALA/Player.py:97-114,176-181; stacked by IMPALA/ReplayMemory.py:34-43).
    -> [state, action, mu, reward, done]  (done keeps the reference's name and meaning: 1 = bootstrap)"""
    n = len(recs)
    s = np.empty((n, T + 1, 4 * 84 * 84), np.uint8)
    a = np.empty((n, T), np.int32)
    mu = np.empty((n, T), np.float32)
    rw = np.empty((n, T), np.float32)
    d = np.empty(n, np.float32)
    for i, r in enumerate(recs):
        s[i] = np.asarray(r[0], np.uint8).reshape(T + 1, -1)
        a[i] = np.asarray(r[1]).reshape(T).astype(np.int32)
        mu[i] = np.asarray(r[2], np.float32).reshape(T)
        rw[i] = np.asarray(r[3], np.float32).reshape(T)
        d[i] = float(r[4])
    return [s, a, mu, rw, d]


# ---------------------------------------------------------------------------------------------
# record templates: the byte layout one actor fleet's pickles share, decoded on the GPU (DESIGN.md §4.24)
# ---------------------------------------------------------------------------------------------
# A template sorts every byte of a record's pickle into skeleton (compared byte for byte), value spans (converted into
# a field of the decoded batch) and free spans (bytes that differ from record to record and carry no value).  Records
# whose skeleton equals the template's are parsed exactly as the template's record was, so the value spans sit at the
# same offsets and mean the same fields: b2rl_wire_decode checks the skeleton and scatters the values.
#
# A run is 8 int32: [op, src, len, field, dst, count, aux, kinds].  src / len: the bytes of the record it covers; field
# / dst: destination field and byte offset within the record's row; kinds = source kind | destination kind << 8.
RUN_SKELETON, RUN_SAME, RUN_COPY, RUN_STRIP, RUN_CONVERT = 0, 1, 2, 3, 4
# RUN_SAME: record bytes [src, src + len) must equal record bytes [aux, aux + len).  RUN_STRIP: stack `count` of an R2D2
# sequence (4 frames at src) into a frame strip; aux = the next stack's offset, or -1 for the last stack.
S_U8, S_U16, S_I32, S_I64, S_F32, S_F64, S_F64BE, S_BOOLOP, S_B1 = range(9)
SRC_BYTES = (1, 2, 4, 8, 4, 8, 8, 1, 1)
SRC_FLOAT = (S_F32, S_F64, S_F64BE)
D_I32, D_F32, D_F32_DIRECT, D_U8_BOOL, D_F32_NOT = range(5)
# D_F32: float(x) then the float32 store (an int rounds to double first, as Python's float() does, and a float32 NaN is
# quieted by the widening); D_F32_DIRECT: numpy's array cast to float32 (an int rounds once, a float32 keeps its bits).
# D_U8_BOOL: bool(x).  D_F32_NOT: float(not x).
STATUS_OK, STATUS_SKELETON, STATUS_RANGE, STATUS_NO_SLIDE = 0, 1, 2, 4
TASK_BYTES = 32 << 10            # record bytes per CTA (runs are whole; a frame stack is never split)
FRAME_BYTES, STACK_BYTES = 84 * 84, 4 * 84 * 84
_TORCH_MAGIC = 0x1950A86A20F9469CFC6C
_NUMPY = ("numpy._core.multiarray", "numpy.core.multiarray")
_NUMERIC = ("numpy._core.numeric", "numpy.core.numeric")
_DTYPE_KIND = {"<f8": S_F64, "<f4": S_F32, "<i8": S_I64, "<i4": S_I32, "|u1": S_U8, "<u2": S_U16, "|b1": S_B1}


class _Unsupported(Exception):
    """Something derivation cannot fully account for: the records take the host path."""


def _need(cond):
    if not cond:
        raise _Unsupported


class _G:
    __slots__ = ("module", "name")

    def __init__(self, module, name):
        self.module, self.name = module, name

    def __eq__(self, other):
        return isinstance(other, _G) and (self.module, self.name) == (other.module, other.name)

    __hash__ = None


class _V:
    """A literal: value, the offset / length of its bytes in the record and its source kind (None: not a value)."""
    __slots__ = ("value", "off", "n", "kind")

    def __init__(self, value, off, n, kind):
        self.value, self.off, self.n, self.kind = value, off, n, kind


class _R:
    """callable(*args), with the state a BUILD gave it."""
    __slots__ = ("fn", "args", "state")

    def __init__(self, fn, args):
        self.fn, self.args, self.state = fn, args, None


_INT_ARGS = {"BININT1": (1, S_U8), "BININT2": (2, S_U16), "BININT": (4, S_I32)}
_BYTES_OPS = ("SHORT_BINBYTES", "BINBYTES", "BINBYTES8", "BYTEARRAY8")
_STR_OPS = ("SHORT_BINUNICODE", "BINUNICODE", "BINUNICODE8")


def _symbolic_load(blob: bytes):
    """The object tree a pickle builds, with every literal kept as a _V at its bytes."""
    import pickletools
    ops = list(pickletools.genops(blob))
    _need(ops and ops[-1][0].name == "STOP" and ops[-1][2] == len(blob) - 1)
    stack, marks, memo = [], [], {}
    for i, (op, arg, pos) in enumerate(ops):
        name, end = op.name, (ops[i + 1][2] if i + 1 < len(ops) else len(blob))
        if name in ("PROTO", "FRAME"):
            continue
        if name == "STOP":
            _need(len(stack) == 1 and not marks)
            return stack[0]
        if name == "MARK":
            marks.append(len(stack))
        elif name in _INT_ARGS:
            n, kind = _INT_ARGS[name]
            stack.append(_V(arg, end - n, n, kind))
        elif name == "LONG1":
            stack.append(_V(arg, pos, end - pos, None))
        elif name == "BINFLOAT":
            stack.append(_V(arg, end - 8, 8, S_F64BE))
        elif name in ("NEWTRUE", "NEWFALSE"):
            stack.append(_V(name == "NEWTRUE", pos, 1, S_BOOLOP))
        elif name == "NONE":
            stack.append(None)
        elif name in _BYTES_OPS:
            stack.append(_V(bytes(arg), end - len(arg), len(arg), None))
        elif name in _STR_OPS:
            stack.append(arg)
        elif name == "EMPTY_LIST":
            stack.append([])
        elif name == "EMPTY_TUPLE":
            stack.append(())
        elif name in ("TUPLE1", "TUPLE2", "TUPLE3"):
            k = int(name[-1])
            _need(len(stack) >= k)
            stack[-k:] = [tuple(stack[-k:])]
        elif name in ("TUPLE", "LIST", "APPENDS"):
            _need(marks)
            at = marks.pop()
            items = stack[at:]
            del stack[at:]
            if name == "APPENDS":
                _need(stack and isinstance(stack[-1], list))
                stack[-1].extend(items)
            else:
                stack.append(tuple(items) if name == "TUPLE" else list(items))
        elif name == "APPEND":
            _need(len(stack) >= 2 and isinstance(stack[-2], list))
            stack[-2].append(stack.pop())
        elif name in ("MEMOIZE", "BINPUT", "LONG_BINPUT"):
            _need(stack)
            memo[len(memo) if name == "MEMOIZE" else arg] = stack[-1]
        elif name in ("BINGET", "LONG_BINGET"):
            _need(arg in memo)
            stack.append(memo[arg])
        elif name == "GLOBAL":
            stack.append(_G(*arg.split(" ", 1)))
        elif name == "STACK_GLOBAL":
            _need(len(stack) >= 2 and isinstance(stack[-2], str) and isinstance(stack[-1], str))
            stack[-2:] = [_G(stack[-2], stack[-1])]
        elif name == "REDUCE":
            _need(len(stack) >= 2 and isinstance(stack[-2], _G) and isinstance(stack[-1], tuple))
            stack[-2:] = [_R(stack[-2], stack[-1])]
        elif name == "BUILD":
            _need(len(stack) >= 2 and isinstance(stack[-2], _R) and stack[-2].state is None)
            state = stack.pop()
            stack[-1].state = state
        else:
            raise _Unsupported
        _need(not marks or marks[-1] <= len(stack))
    raise _Unsupported


def _lit(x, types):
    """The value of a skeleton literal (it is part of the template, so every matching record has it too)."""
    v = x.value if isinstance(x, _V) else x
    _need(isinstance(v, types) and (types is bool) == isinstance(v, bool))
    return v


def _dtype(node) -> str:
    _need(isinstance(node, _R) and node.fn == _G("numpy", "dtype") and len(node.args) == 3)
    name = _lit(node.args[0], str)
    _need(_lit(node.args[1], bool) is False and _lit(node.args[2], bool) is True)
    st = node.state
    _need(isinstance(st, tuple) and len(st) == 8 and _lit(st[0], int) == 3 and st[2:5] == (None, None, None)
          and [_lit(x, int) for x in st[5:7]] == [-1, -1] and _lit(st[7], int) in (0, 63))
    order = _lit(st[1], str)
    _need(order in ("<", "|", "="))
    return ("|" if order == "|" else "<") + name


def _shape(t) -> tuple:
    _need(isinstance(t, tuple))
    return tuple(_lit(x, int) for x in t)


def _ndarray(node):
    """-> (dtype str, shape, payload _V, or the item list of an object array)."""
    _need(isinstance(node, _R) and isinstance(node.fn, _G))
    if node.fn.module in _NUMPY and node.fn.name == "_reconstruct":
        _need(len(node.args) == 3 and node.args[0] == _G("numpy", "ndarray") and _shape(node.args[1]) == (0,)
              and _lit(node.args[2], bytes) == b"b")
        st = node.state
        _need(isinstance(st, tuple) and len(st) == 5 and _lit(st[0], int) == 1 and _lit(st[3], bool) is False)
        dt, shape, data = _dtype(st[2]), _shape(st[1]), st[4]
    elif node.fn.module in _NUMERIC and node.fn.name == "_frombuffer":
        _need(len(node.args) == 4 and node.state is None and _lit(node.args[3], str) == "C")
        dt, shape, data = _dtype(node.args[1]), _shape(node.args[2]), node.args[0]
    else:
        raise _Unsupported
    numel = int(np.prod(shape, dtype=np.int64))
    if dt == "|O8":
        _need(isinstance(data, list) and len(data) == numel)
    else:
        _need(dt in _DTYPE_KIND and isinstance(data, _V) and isinstance(data.value, bytes)
              and data.n == numel * SRC_BYTES[_DTYPE_KIND[dt]])
    return dt, shape, data


def _scalar(node) -> tuple:
    """A Python int / float / bool or a numpy scalar -> (source kind, offset)."""
    if isinstance(node, _V):
        _need(node.kind is not None)
        return node.kind, node.off
    _need(isinstance(node, _R) and isinstance(node.fn, _G) and node.fn.module in _NUMPY and node.fn.name == "scalar"
          and node.state is None and len(node.args) == 2)
    dt, data = _dtype(node.args[0]), node.args[1]
    _need(dt in _DTYPE_KIND and isinstance(data, _V) and isinstance(data.value, bytes)
          and data.n == SRC_BYTES[_DTYPE_KIND[dt]])
    return _DTYPE_KIND[dt], data.off


class _Builder:
    """Collects a template's runs and the spans they cover."""

    def __init__(self, fields):
        self.fields = [f[0] for f in fields]
        self.runs, self.covered, self.free_spans = [], [], []

    def run(self, op, src, n, field=0, dst=0, count=0, aux=0, kinds=0):
        self.runs.append((op, src, n, self.fields.index(field) if isinstance(field, str) else field, dst, count, aux,
                          kinds))
        self.covered.append((src, n))

    def free(self, src, n):
        self.covered.append((src, n))
        self.free_spans.append((src, n))

    def scalar(self, node, field, dst, to):
        kind, off = _scalar(node)
        _need(to != D_I32 or kind not in SRC_FLOAT)
        self.run(RUN_CONVERT, off, SRC_BYTES[kind], field, dst, 1, 0, kind | to << 8)

    def array(self, node, field, numel, to):
        """A numeric array of `numel` elements converted element by element into float32 / int32."""
        dt, _, data = _ndarray(node)
        _need(dt != "|O8" and data.n // SRC_BYTES[_DTYPE_KIND[dt]] == numel)
        kind = _DTYPE_KIND[dt]
        if to == D_I32:
            _need(kind not in SRC_FLOAT and kind != S_B1)
        else:
            to = D_F32_DIRECT            # np.asarray(x, np.float32) / astype: a float32 NaN keeps its bits
        self.run(RUN_CONVERT, data.off, data.n, field, 0, numel, 0, kind | to << 8)

    def frames(self, node, numel) -> int:
        """A uint8 array of `numel` elements -> the offset of its payload."""
        dt, _, data = _ndarray(node)
        _need(dt == "|u1" and data.n == numel)
        return data.off

    def hidden(self, node, field, hidden):
        """An LSTM state, a torch tensor or a numpy array of `hidden` values -> float32 (wire._hidden)."""
        if isinstance(node, _R) and node.fn == _G("torch._utils", "_rebuild_tensor_v2"):
            _need(node.state is None and len(node.args) == 6)
            storage, offset, size, stride, grad, hooks = node.args
            _need(_lit(offset, int) == 0 and _lit(grad, bool) is False)
            size, stride = _shape(size), _shape(stride)
            _need(int(np.prod(size)) == hidden and stride == tuple(int(np.prod(size[i + 1:])) for i in range(len(size))))
            _need(isinstance(hooks, _R) and hooks.fn == _G("collections", "OrderedDict") and hooks.args == ()
                  and hooks.state is None)
            _need(isinstance(storage, _R) and storage.fn == _G("torch.storage", "_load_from_bytes")
                  and storage.state is None and len(storage.args) == 1)
            data = storage.args[0]
            _need(isinstance(data, _V) and isinstance(data.value, bytes))
            self._torch_storage(data, field, hidden)
            return
        self.array(node, field, hidden, D_F32)

    def _torch_storage(self, data: _V, field, hidden):
        """torch.save's legacy format inside a pickled storage: magic number, protocol, system info, the storage's
        persistent id, its key list, then the element count and the raw little-endian elements.  The storage key
        (a number torch derives from the storage's address) is free where it first appears; the key list must repeat
        it (RUN_SAME).  Everything else is skeleton."""
        import io
        import pickletools
        raw, base = data.value, data.off
        f = io.BytesIO(raw)
        parts = []
        for _ in range(5):
            start = f.tell()
            parts.append([(op.name, arg, pos) for op, arg, pos in pickletools.genops(f)])
            parts[-1].append(("END", None, f.tell()))
            _need(parts[-1][0][0] == "PROTO")
            del start
        _need([o for o, _, _ in parts[0]] == ["PROTO", "LONG1", "STOP", "END"] and parts[0][1][1] == _TORCH_MAGIC)
        _need([o for o, _, _ in parts[1]] == ["PROTO", "BININT2", "STOP", "END"] and parts[1][1][1] == 1001)
        s, e = parts[2][0][2], parts[2][-1][2]
        info = pickle.loads(raw[s:e])
        _need(isinstance(info, dict) and info.get("little_endian") is True)
        pid = parts[3]
        _need([o for o, _, _ in pid[:2]] == ["PROTO", "MARK"] and pid[2][:2] == ("BINUNICODE", "storage")
              and pid[4][:2] == ("GLOBAL", "torch FloatStorage") and pid[6][0] == "BINUNICODE"
              and pid[8][:2] == ("BINUNICODE", "cpu") and pid[10][0] in _INT_ARGS
              and [o for o, _, _ in pid[11:]] == ["NONE", "TUPLE", "BINPUT", "BINPERSID", "STOP", "END"]
              and all(pid[k][0] == "BINPUT" for k in (3, 5, 7, 9)))
        key, numel = pid[6][1], pid[10][1]
        _need(key.isascii() and key.isdigit() and numel == hidden)
        keys = parts[4]
        _need([o for o, _, _ in keys] == ["PROTO", "EMPTY_LIST", "BINPUT", "BINUNICODE", "BINPUT", "APPEND", "STOP",
                                          "END"] and keys[3][1] == key)
        key_at, again_at = pid[7][2] - len(key), keys[4][2] - len(key)
        self.free(base + key_at, len(key))
        self.run(RUN_SAME, base + again_at, len(key), aux=base + key_at)
        at = keys[-1][2]
        _need(int.from_bytes(raw[at:at + 8], "little") == numel and len(raw) == at + 8 + 4 * numel)
        self.run(RUN_CONVERT, base + at + 8, 4 * numel, field, 0, numel, 0, S_F32 | D_F32_DIRECT << 8)


class Template:
    """The byte layout of one kind of record: `blob` (the record it was derived from, whose skeleton bytes every
    matching record repeats), `runs` (int32 (R, 8)), `tasks` (int32 (K, 2): the runs of each CTA), `free` (the
    (offset, length) spans no run reads), `fields` (the decoded batch's (name, dtype, per-record shape) in order) and
    `digest` (of the skeleton and the runs)."""

    def __init__(self, kind, blob, b: _Builder, fields):
        self.kind, self.blob, self.length, self.fields = kind, bytes(blob), len(blob), tuple(fields)
        self.free = tuple(b.free_spans)
        cover = np.zeros(len(blob) + 1, np.int32)
        for s, n in b.covered:
            cover[s] += 1
            cover[s + n] -= 1
        skel = np.cumsum(cover[:-1]) == 0
        edges = np.flatnonzero(np.diff(np.concatenate(([0], skel.astype(np.int8), [0]))))
        runs = [(RUN_SKELETON, int(s), int(e - s), 0, 0, 0, 0, 0) for s, e in zip(edges[::2], edges[1::2])]
        runs = sorted(runs + b.runs, key=lambda r: (r[1], r[0]))
        self.runs = np.asarray(runs, np.int32).reshape(-1, 8)
        self.skeleton = skel
        tasks, start, acc = [], 0, 0
        for i, r in enumerate(runs):
            acc += r[2]
            if acc >= TASK_BYTES:
                tasks.append((start, i + 1))
                start, acc = i + 1, 0
        if start < len(runs):
            tasks.append((start, len(runs)))
        self.tasks = np.asarray(tasks, np.int32).reshape(-1, 2)
        import hashlib
        h = hashlib.blake2b(digest_size=16)
        h.update(np.frombuffer(self.blob, np.uint8)[skel].tobytes())
        h.update(self.runs.tobytes())
        self.digest = h.digest()


def record_fields(kind: str, T: int = 0, hidden: int = 512, strip: bool = False) -> tuple:
    """The decoded batch of one record kind: (name, numpy dtype, per-record shape), the host decoders' layout."""
    u8, i32, f32 = np.uint8, np.int32, np.float32
    if kind == "apex":
        return (("s", u8, (4, 84, 84)), ("ns", u8, (4, 84, 84)), ("a", i32, ()), ("r", f32, ()), ("d", u8, ()),
                ("p", f32, ()))
    if kind == "r2d2":
        return (("state", u8, (T + 3, 84, 84) if strip else (T, 4, 84, 84)), ("action", i32, (T,)),
                ("reward", f32, (T,)), ("h0", f32, (hidden,)), ("h1", f32, (hidden,)), ("notdone", f32, ()),
                ("p", f32, ()))
    if kind == "impala":
        return (("state", u8, (T + 1, STACK_BYTES)), ("action", i32, (T,)), ("mu", f32, (T,)), ("reward", f32, (T,)),
                ("done", f32, ()))
    raise ValueError(f"unknown record kind {kind!r}")


def derive_template(blob: bytes, kind: str, T: int = 0, hidden: int = 512, strip: bool = False):
    """The Template of `blob`, a pickled record of `kind` ("apex", "r2d2", "impala"), or None when derivation meets
    anything it cannot fully account for (such records are decoded on the host)."""
    fields = record_fields(kind, T, hidden, strip)
    b = _Builder(fields)
    try:
        root = _symbolic_load(bytes(blob))
        if kind == "apex":
            _need(isinstance(root, list) and len(root) == 6)
            b.run(RUN_COPY, b.frames(root[0], STACK_BYTES), STACK_BYTES, "s")
            b.run(RUN_COPY, b.frames(root[3], STACK_BYTES), STACK_BYTES, "ns")
            b.scalar(root[1], "a", 0, D_I32)
            b.scalar(root[2], "r", 0, D_F32)
            b.scalar(root[4], "d", 0, D_U8_BOOL)
            b.scalar(root[5], "p", 0, D_F32)
        elif kind == "r2d2":
            if isinstance(root, _R):
                dt, shape, items = _ndarray(root)
                _need(dt == "|O8" and len(shape) == 1)
            else:
                items = root
            _need(isinstance(items, list) and len(items) == 3 * T + 3 and T > 0)
            _need(isinstance(items[0], tuple) and len(items[0]) == 2)
            b.hidden(items[0][0], "h0", hidden)
            b.hidden(items[0][1], "h1", hidden)
            stacks = [b.frames(items[1 + 3 * t], STACK_BYTES) for t in range(T)]
            for t in range(T):
                if strip:
                    b.run(RUN_STRIP, stacks[t], STACK_BYTES, "state", 0, t, stacks[t + 1] if t + 1 < T else -1)
                else:
                    b.run(RUN_COPY, stacks[t], STACK_BYTES, "state", t * STACK_BYTES)
                b.scalar(items[2 + 3 * t], "action", 4 * t, D_I32)
                b.scalar(items[3 + 3 * t], "reward", 4 * t, D_F32)
            b.scalar(items[-2], "notdone", 0, D_F32_NOT)
            b.scalar(items[-1], "p", 0, D_F32)
        elif kind == "impala":
            _need(isinstance(root, list) and len(root) == 5 and T > 0)
            b.run(RUN_COPY, b.frames(root[0], (T + 1) * STACK_BYTES), (T + 1) * STACK_BYTES, "state")
            b.array(root[1], "action", T, D_I32)
            b.array(root[2], "mu", T, D_F32)
            b.array(root[3], "reward", T, D_F32)
            b.scalar(root[4], "done", 0, D_F32)
        else:
            raise ValueError(f"unknown record kind {kind!r}")
    except (_Unsupported, ValueError, TypeError, IndexError, KeyError, EOFError, pickle.UnpicklingError):
        if kind not in ("apex", "r2d2", "impala"):
            raise
        return None
    return Template(kind, blob, b, fields)


class WireIngest:
    """Lists of pickled records of one kind -> a device batch in the host decoders' layout (record_fields), decoded
    by b2rl_wire_decode on a stream of its own.

    The blobs are grouped by template (looked up by length; derived from the first blob of a new length), packed into
    one pinned staging buffer by b2rl_wire_gather and copied to the device once; each group is one launch.  The only
    synchronisation, reading the status words, waits on this stream alone, never behind a learner's queued steps.
    Records without a template, or whose status is not ok, are decoded on the host (decode_apex / decode_r2d2 /
    decode_impala) into their rows of the batch, so the batch holds the records in list order."""

    MAX_TEMPLATES = 8

    def __init__(self, kind: str, device, T: int = 0, hidden: int = 512, strip: bool = False):
        self.kind, self.T, self.hidden, self.strip = kind, T, hidden, strip
        self.device = torch.device(device)
        self.fields = record_fields(kind, T, hidden, strip)
        self.lib = self.stream = None          # made by the first decode
        self.templates = []          # (Template, its device bytes, runs, tasks), most recently added first
        self._stage = self._status = None
        self.host_records = 0        # records decoded on the host so far (no template, or a status that is not ok)

    def _template(self, length: int):
        for t in self.templates:
            if t[0].length == length:
                return t
        return None

    def _add(self, tp: Template):
        for t in self.templates:
            if t[0].digest == tp.digest and t[0].length == tp.length:
                return t
        with torch.cuda.stream(self.stream):
            dev = tuple(torch.from_numpy(np.ascontiguousarray(x)).to(self.device) for x in
                        (np.frombuffer(bytearray(tp.blob), np.uint8), tp.runs, tp.tasks))
        entry = (tp,) + dev
        self.templates = [entry] + self.templates[:self.MAX_TEMPLATES - 1]
        return entry

    def _derive(self, blob):
        tp = derive_template(blob, self.kind, self.T, self.hidden, self.strip)
        return None if tp is None else self._add(tp)

    def _pinned(self, attr: str, n: int, dtype) -> torch.Tensor:
        from .hostmem import pinned_empty
        t = getattr(self, attr)
        if t is None or t.numel() < n:
            t = pinned_empty((max(n, 2 * (t.numel() if t is not None else 0)),), dtype, self.device)
            setattr(self, attr, t)
        return t

    def _host_rows(self, recs) -> list:
        if self.kind == "apex":
            out = {name: np.empty((len(recs),) + shape, dt) for name, dt, shape in self.fields}
            decode_apex(recs, out)
            return [out[name] for name, _, _ in self.fields]
        if self.kind == "r2d2":
            cols, p = decode_r2d2(recs, self.T, self.hidden, self.strip)
            return cols + [p]
        return decode_impala(recs, self.T)

    def decode(self, blobs) -> dict | None:
        """-> {field name: (n, *shape) device tensor}, ready on the caller's current stream; None when the batch must
        take the host path whole: an R2D2 strip that does not slide, or a record the host decoders refuse (the host
        path then raises today's error, naming the record, with nothing pushed); and always for a device that is not
        a GPU."""
        import ctypes as C
        from . import _lib
        from ._lib import check
        if self.device.type != "cuda":
            return None
        if self.stream is None:
            self.lib, self.stream = _lib.load(), torch.cuda.Stream(self.device)
        blobs = [b if isinstance(b, bytes) else bytes(b) for b in blobs]
        n = len(blobs)
        groups, host, tried = {}, [], set()
        for i, b in enumerate(blobs):
            t = self._template(len(b))
            if t is None and len(b) not in tried:
                tried.add(len(b))
                t = self._derive(b)
            if t is None:
                host.append(i)
            else:
                groups.setdefault(id(t), (t, []))[1].append(i)
        plan, total = [], 0
        for t, pos in groups.values():
            stride = (t[0].length + 16 + 15) // 16 * 16
            plan.append((t, pos, total, stride))
            total += len(pos) * stride
        stage = self._pinned("_stage", total + 8 * n, torch.uint8)
        status_h = self._pinned("_status", n, torch.int32)
        base = stage.data_ptr()
        k = 0
        for t, pos, off, stride in plan:
            src = (C.c_char_p * len(pos))(*[blobs[i] for i in pos])
            ln = np.fromiter((len(blobs[i]) for i in pos), np.int64, len(pos))
            check(self.lib.b2rl_wire_gather(src, ln.ctypes.data_as(C.POINTER(C.c_int64)), len(pos), base + off,
                                            stride, base + total + 4 * k))
            k += len(pos)
        rows_h = np.frombuffer(stage.numpy(), np.int32, k, total + 4 * n) if k else None
        if k:
            rows_h[:] = [i for _, pos, _, _ in plan for i in pos]
        out = {}
        with torch.cuda.stream(self.stream):
            for name, dt, shape in self.fields:
                out[name] = torch.empty((n,) + shape, dtype=getattr(torch, np.dtype(dt).name), device=self.device)
            status = torch.zeros(n, dtype=torch.int32, device=self.device)
            if k:
                dev = stage[:total + 8 * n].to(self.device, non_blocking=True)
                ptrs = (C.c_void_p * len(self.fields))(*[out[name].data_ptr() for name, _, _ in self.fields])
                row_bytes = (C.c_int64 * len(self.fields))(*[out[name][0].numel() * out[name].element_size()
                                                             for name, _, _ in self.fields])
                k = 0
                for t, pos, off, stride in plan:
                    tp, tbytes, truns, ttasks = t
                    check(self.lib.b2rl_wire_decode(
                        dev.data_ptr() + off, stride, dev.data_ptr() + total + 4 * k, len(pos), tbytes.data_ptr(),
                        tp.length, truns.data_ptr(), len(tp.runs), ttasks.data_ptr(), len(tp.tasks),
                        dev.data_ptr() + total + 4 * n + 4 * k, ptrs, row_bytes, len(self.fields), status.data_ptr(),
                        n, self.stream.cuda_stream))
                    k += len(pos)
                status_h[:n].copy_(status, non_blocking=True)
                self.stream.synchronize()
            st = status_h[:n].numpy()
            if (st & STATUS_NO_SLIDE).any():
                return None
            bad = np.flatnonzero(st != STATUS_OK)
            for i in bad[:1]:
                if st[i] & STATUS_SKELETON and len(blobs[i]) not in tried:      # a new layout of a known length
                    self._derive(blobs[i])
            fallback = sorted(host + bad.tolist())
            if fallback:
                try:
                    cols = self._host_rows([pickle.loads(blobs[i]) for i in fallback])
                except Exception:
                    return None
                idx = torch.as_tensor(fallback, dtype=torch.int64).to(self.device)
                for (name, _, _), x in zip(self.fields, cols):
                    out[name].index_copy_(0, idx, torch.from_numpy(np.ascontiguousarray(x)).to(self.device))
                self.host_records += len(fallback)
        cur = torch.cuda.current_stream(self.device)
        cur.wait_stream(self.stream)
        for t in out.values():
            t.record_stream(cur)
        return out
