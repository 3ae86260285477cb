"""In-tree build of libb2rl.so (the C-ABI CUDA library) with nvcc for sm_90a (H100).

    python -m distributed_rl_b200.build        # (re)build if sources are newer

nvcc cross-compiles without a GPU; the built .so is git-ignored and lives next to
this file, so the package is importable straight from the source tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb2rl.so")
STAMP = LIB + ".stamp"     # the nvcc flags the library was built with: a change of target or flags forces a rebuild
SOURCES = ["capi.cu", "tree.cu", "gather.cu", "targets.cu", "conv1.cu", "conv1_wgrad.cu", "optim.cu", "gemm.cu", "dueling.cu", "peer.cu", "serve.cu",
           "uniform.cu", "dedup.cu", "hostrows.cu", "wire.cu", "stem.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false",            # every fp op individually rounded (parity with the numpy oracle)
    "-Xcompiler", "-fPIC", "-shared",
    "-diag-suppress", "177",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found (looked at $NVCC, PATH, /usr/local/cuda/bin/nvcc)")


def sources() -> list[str]:
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.isfile(os.path.join(CSRC, s))]


def _flags_id() -> str:
    return " ".join(NVCC_FLAGS) + "\n"


def needs_build() -> bool:
    if not os.path.isfile(LIB) or not os.path.isfile(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != _flags_id():
            return True
    t = os.path.getmtime(LIB)
    deps = sources() + [os.path.join(CSRC, "common.cuh"),
                        os.path.join(os.path.dirname(HERE), "include", "b2rl.h")]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.isfile(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + sources()
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    with open(STAMP, "w") as f:
        f.write(_flags_id())
    if verbose:
        print(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
