"""Pinned host staging for the ingest path, allocated on the GPU's NUMA node when it is known.

The replay server feeds the learner from host memory (decoded Redis records,
APE_X/ReplayMemory.py:128-139).  Staging buffers are pinned so the H2D copy is a straight DMA that
overlaps the learner step.  cudaHostAlloc places pages on the node of the allocating thread, so the
buffers are allocated with the thread temporarily bound to the GPU's node (best effort; a no-op when
sysfs does not expose the topology).  The binding is a safeguard for hosts with a slow socket
interconnect, not a measured win (tools/h2d_probe.py measures the copy rate from each node).
"""
from __future__ import annotations

import contextlib
import os

import torch


def _parse_cpulist(s: str) -> set[int]:
    out: set[int] = set()
    for part in s.strip().split(","):
        if "-" in part:
            a, b = part.split("-")
            out |= set(range(int(a), int(b) + 1))
        elif part:
            out.add(int(part))
    return out


def gpu_node_cpus(device) -> set[int] | None:
    """CPUs of the NUMA node the GPU hangs off, or None when the topology is not exposed."""
    try:
        p = torch.cuda.get_device_properties(torch.device(device))
        name = f"{getattr(p, 'pci_domain_id', 0):04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{name}/numa_node") as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = _parse_cpulist(f.read())
        return cpus or None
    except (OSError, ValueError, AttributeError, RuntimeError):
        return None


@contextlib.contextmanager
def on_gpu_node(device):
    """Bind the calling thread to the GPU's NUMA node for the duration (no-op if unknown)."""
    cpus = gpu_node_cpus(device)
    if not cpus or not hasattr(os, "sched_setaffinity"):
        yield False
        return
    old = os.sched_getaffinity(0)
    target = (cpus & old) or cpus
    try:
        os.sched_setaffinity(0, target)
    except OSError:
        yield False
        return
    try:
        yield True
    finally:
        os.sched_setaffinity(0, old)


def pinned_empty(shape, dtype, device) -> torch.Tensor:
    """Pinned host tensor whose pages sit on the NUMA node of `device`."""
    with on_gpu_node(device):
        t = torch.empty(shape, dtype=dtype, pin_memory=True)
        t.view(torch.uint8).zero_() if t.numel() else None      # touch on this node
    return t


def pinned_like(x, device) -> torch.Tensor:
    """Pinned copy of a host tensor / ndarray on the NUMA node of `device`."""
    x = torch.as_tensor(x)
    t = pinned_empty(x.shape, x.dtype, device)
    t.copy_(x)
    return t
