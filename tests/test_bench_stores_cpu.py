"""tools/bench_stores.py without a GPU: every store form in its table builds a learner config that passes the config's
own checks, and its command line refuses what it documents refusing."""
import importlib.util
import os
import subprocess
import sys

import pytest

SCRIPT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "bench_stores.py")


def _load():
    spec = importlib.util.spec_from_file_location("bench_stores", SCRIPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


bs = _load()


@pytest.mark.parametrize("workload,form", [(w, f) for w in bs.STORES for f in bs.STORES[w]])
def test_every_store_form_builds_its_config(workload, form):
    cfg = bs.config(workload, form, bs.DEFAULTS[workload]["slots"], bs.DEFAULTS[workload]["batch"][0])
    for key, value in bs.STORES[workload][form].items():
        assert getattr(cfg, key) == value
    cfg.__post_init__()
    assert bs.dedup(workload, form) == bool(getattr(cfg, "FRAME_DEDUP", False))
    if bs.dedup(workload, form):
        bs.MODULES[workload].dedup_geometry(cfg)
    if bs.coded(workload, form):
        assert bs.MODULES[workload].pool_bytes(cfg) > 0


def test_host_stores_count_their_pinned_bytes():
    slots = 1 << 10
    assert bs.host_bytes("r2d2", bs.config("r2d2", "host_frames", slots)) == slots * bs.STRIP_BYTES
    cfg = bs.config("r2d2", "host_pool", slots)
    assert bs.host_bytes("r2d2", cfg) == bs.r2d2.dedup_geometry(cfg)[0] * bs.R.FRAME_BYTES
    assert all(bs.host_bytes(w, bs.config(w, f, slots)) == 0 for w in bs.STORES for f in bs.STORES[w]
               if f not in ("host_frames", "host_pool"))


def test_default_measurements_follow_the_stores():
    assert bs.parse(["--workload", "apex", "--stores", "stacks", "dedup"]).measure == [
        "bytes", "push", "step", "served", "capacity", "kernels"]
    assert bs.parse(["--workload", "r2d2", "--stores", "strips"]).measure == [
        "bytes", "push", "step", "served", "capacity"]
    assert "staging" in bs.parse(["--workload", "impala", "--stores", "dedup", "coded"]).measure


def _run(*args):
    return subprocess.run([sys.executable, SCRIPT, *args], capture_output=True, text=True, timeout=300)


def test_help():
    p = _run("--help")
    assert p.returncode == 0
    assert "--workload" in p.stdout and "--stores" in p.stdout and "--measure" in p.stdout


@pytest.mark.parametrize("args,message", [
    (("--workload", "r2d2", "--stores", "strips", "pool"), "unknown r2d2 store pool"),
    (("--workload", "apex", "--stores", "strips"), "unknown apex store strips"),
    (("--workload", "r2d2", "--stores", "dedup", "--measure", "kernels"), "kernels does not apply to r2d2 dedup"),
])
def test_refused_command_lines(args, message):
    p = _run(*args)
    assert p.returncode == 2
    assert message in p.stderr
