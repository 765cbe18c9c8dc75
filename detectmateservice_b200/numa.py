"""NUMA placement of pinned host buffers.

A pinned buffer lives on the NUMA node of the thread that allocated it; when that is not the
node the GPU's PCIe root hangs off, host -> device copies can run well below the link rate.
`bound_to_gpu_node(device)` pins the calling thread to the GPU-local CPUs while the buffers
are allocated (and first touched) and restores the affinity afterwards.  Pure host-side
plumbing around the boundary; nothing here computes.
"""
from __future__ import annotations

import contextlib
import os
from typing import Optional, Set


def parse_cpulist(text: str) -> Set[int]:
    """'0-3,8,10-11' -> {0,1,2,3,8,10,11} (the format of /sys/devices/system/node/nodeN/cpulist)."""
    cpus: Set[int] = set()
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            lo, hi = part.split("-", 1)
            cpus.update(range(int(lo), int(hi) + 1))
        else:
            cpus.add(int(part))
    return cpus


def gpu_numa_cpus(device: int = 0, sysfs: str = "/sys") -> Optional[Set[int]]:
    """CPUs of the NUMA node the CUDA device `device` is attached to, None if unknown."""
    try:
        import torch
        p = torch.cuda.get_device_properties(device)
        bdf = "%04x:%02x:%02x.0" % (getattr(p, "pci_domain_id", 0), p.pci_bus_id, p.pci_device_id)
        with open(os.path.join(sysfs, "bus/pci/devices", bdf, "numa_node")) as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open(os.path.join(sysfs, "devices/system/node/node%d/cpulist" % node)) as f:
            cpus = parse_cpulist(f.read())
        allowed = os.sched_getaffinity(0)
        cpus &= allowed
        return cpus or None
    except Exception:
        return None


def gpu_numa_node(device: int = 0, sysfs: str = "/sys") -> Optional[int]:
    try:
        import torch
        p = torch.cuda.get_device_properties(device)
        bdf = "%04x:%02x:%02x.0" % (getattr(p, "pci_domain_id", 0), p.pci_bus_id, p.pci_device_id)
        with open(os.path.join(sysfs, "bus/pci/devices", bdf, "numa_node")) as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except Exception:
        return None


_SYS_SET_MEMPOLICY = 238          # x86_64
_MPOL_DEFAULT, _MPOL_PREFERRED = 0, 1


def _set_mempolicy(mode: int, node: Optional[int]) -> bool:
    """set_mempolicy(2) for the calling thread: where the kernel takes the pages of the
    allocations it makes on this thread's behalf (cudaHostAlloc included)."""
    import ctypes
    import platform
    if platform.machine() != "x86_64":
        return False
    try:
        libc = ctypes.CDLL(None, use_errno=True)
        if node is None:
            rc = libc.syscall(_SYS_SET_MEMPOLICY, mode, None, 0)
        else:
            mask = (ctypes.c_ulong * 16)()
            mask[node // 64] = 1 << (node % 64)
            rc = libc.syscall(_SYS_SET_MEMPOLICY, mode, mask, 16 * 64 + 1)
        return rc == 0
    except Exception:
        return False


@contextlib.contextmanager
def bound_to_gpu_node(device: int = 0):
    """Run the body with the calling thread bound to the GPU's NUMA node: memory policy
    MPOL_PREFERRED for that node (what decides where pinned pages come from) and CPU affinity to its
    cores (first touch).  Everything is restored afterwards; a no-op when the topology cannot
    be read.  Yields the CPU set used, or None."""
    cpus = gpu_numa_cpus(device)
    node = gpu_numa_node(device)
    old = None
    policy = False
    if cpus:
        try:
            old = os.sched_getaffinity(0)
            os.sched_setaffinity(0, cpus)
        except OSError:
            old, cpus = None, None
    if node is not None:
        policy = _set_mempolicy(_MPOL_PREFERRED, node)   # preferred, not strict: falls back if the node is full
    try:
        yield cpus
    finally:
        if policy:
            _set_mempolicy(_MPOL_DEFAULT, None)
        if old is not None:
            try:
                os.sched_setaffinity(0, old)
            except OSError:
                pass
