"""CPU-side checks of the C-ABI boundary: the library builds (nvcc cross-compiles
without a GPU), loads, and exports every symbol include/b2rl.h declares — no
compute calls here."""
import ctypes
import os
import re

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(REPO, "include", "b2rl.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2rl_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from distributed_rl_b200 import build, _lib
    build.build()
    return _lib.load()


def test_header_declares_expected_surface():
    syms = _declared_symbols()
    for must in ("b2rl_replay_create", "b2rl_replay_push", "b2rl_tree_sample", "b2rl_tree_update",
                 "b2rl_replay_gather", "b2rl_apex_target", "b2rl_r2d2_target", "b2rl_vtrace"):
        assert must in syms


def test_library_exports_every_declared_symbol(lib):
    from distributed_rl_b200 import _lib
    for s in _declared_symbols():
        assert hasattr(lib, s), f"libb2rl.so does not export {s}"
        assert s in _lib.SIGNATURES, f"ctypes binding missing for {s}"
    assert set(_lib.SIGNATURES) == set(_declared_symbols())


def test_version_and_error_string(lib):
    assert lib.b2rl_version() >= 100
    assert isinstance(lib.b2rl_last_error(), bytes)
    assert lib.b2rl_launch_count() >= 0


def test_invalid_arguments_are_reported_not_crashed(lib):
    from distributed_rl_b200._lib import ReplayDesc
    # null pointers are rejected before any CUDA call
    assert lib.b2rl_replay_create(None, None) < 0
    assert b"null" in lib.b2rl_last_error()
    d = ReplayDesc(); d.capacity = 0; d.n_fields = 0; d.device = 0
    h = ctypes.c_void_p()
    assert lib.b2rl_replay_create(ctypes.byref(d), ctypes.byref(h)) < 0
    assert lib.b2rl_apex_target(*([None] * 7), 0, 0, 0.0, 0.0, *([None] * 6)) < 0
    # the stored-level read-back refuses a null handle or a null n_nodes before it looks at the tree (a level
    # outside 0..G is refused on a live handle: tests/test_gpu_30_tree_at_scale.py)
    n, g, tb = ctypes.c_int64(-1), ctypes.c_int32(-1), ctypes.c_int32(-1)
    for k in (0, 1, -1, 99):
        assert lib.b2rl_tree_level(None, k, ctypes.byref(n), ctypes.byref(g), ctypes.byref(tb), None, None, None) < 0
        assert b"null handle" in lib.b2rl_last_error()
        assert lib.b2rl_tree_level(None, k, None, None, None, None, None, None) < 0
    assert (n.value, g.value, tb.value) == (-1, -1, -1)      # nothing written on a refusal


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from distributed_rl_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.B2RLError, match="no CPU fallback"):
        _lib.load()


def test_device_replay_refuses_cpu_device(lib):
    import torch
    from distributed_rl_b200 import replay
    from distributed_rl_b200._lib import B2RLError
    if torch.cuda.is_available():
        pytest.skip("GPU present; covered by the gpu tests")
    with pytest.raises((B2RLError, RuntimeError, AssertionError)):
        replay.DeviceReplay(16, fields=(), device="cpu")


def _prototypes():
    """name -> list of parameter declarations, parsed from include/b2rl.h."""
    src = open(os.path.join(REPO, "include", "b2rl.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(b2rl_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        params = [p.strip() for p in m.group(2).replace("\n", " ").split(",")]
        protos[m.group(1)] = [] if params in ([""], ["void"]) else params
    return protos


def test_ctypes_signatures_match_the_header_prototypes():
    """Every binding has as many arguments as the prototype, pointers bound as pointers, 64-bit integers and
    doubles with their own width (a mismatch here is silent memory corruption at call time)."""
    from distributed_rl_b200 import _lib
    protos = _prototypes()
    assert set(protos) == set(_lib.SIGNATURES)
    for name, (res, args) in _lib.SIGNATURES.items():
        decl = protos[name]
        assert len(args) == len(decl), f"{name}: {len(args)} ctypes arguments vs {len(decl)} in the header: {decl}"
        for a, d in zip(args, decl):
            is_ptr = "*" in d or d.startswith("void* ") or "b2rl_replay*" in d
            if is_ptr:
                assert a is ctypes.c_void_p or a is ctypes.c_char_p or hasattr(a, "contents") or \
                    getattr(a, "_type_", None) is not None, f"{name}: `{d}` must be bound as a pointer, got {a}"
            elif d.startswith("int64_t"):
                assert a is ctypes.c_int64, f"{name}: `{d}` bound as {a}"
            elif d.startswith("int32_t") or d.startswith("int "):
                assert a in (ctypes.c_int32, ctypes.c_int), f"{name}: `{d}` bound as {a}"
            elif d.startswith("uint64_t"):
                assert a is ctypes.c_uint64, f"{name}: `{d}` bound as {a}"
            elif d.startswith("uint32_t"):
                assert a is ctypes.c_uint32, f"{name}: `{d}` bound as {a}"
            elif d.startswith("double"):
                assert a is ctypes.c_double, f"{name}: `{d}` bound as {a}"
            elif d.startswith("float"):
                assert a is ctypes.c_float, f"{name}: `{d}` bound as {a}"


def test_every_entry_point_cites_the_reference_interface_it_replaces():
    """include/b2rl.h: each declaration is preceded (within its comment block) by a reference file:line citation."""
    src = open(os.path.join(REPO, "include", "b2rl.h")).read()
    blocks = re.split(r"(?=/\*)", src)
    cited = set()
    for b in blocks:
        names = re.findall(r"\b(b2rl_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", b, flags=re.S))
        comment = "".join(re.findall(r"/\*.*?\*/", b, flags=re.S))
        if re.search(r"[A-Za-z_/0-9]+\.(py|json):\d+", comment):
            cited.update(names)
    missing = sorted(set(_declared_symbols()) - cited - {"b2rl_version", "b2rl_last_error", "b2rl_launch_count"})
    assert not missing, f"entry points without a reference citation in their comment: {missing}"
