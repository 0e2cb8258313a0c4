"""NUMA-aware pinned staging buffers for the host -> device leg of the head's inputs.

On a multi-socket host the H2D rate of one step's inputs (8.4 MB of bf16 RoI features) depends on where the pinned
pages live and which cores last wrote them.  ``pinned_like`` allocates and first-touches the staging buffer from ONE thread
bound to the GPU's own NUMA node (``/sys/bus/pci/devices/<bdf>/local_cpulist``), which is what a data-loader
worker pinned next to its GPU would do.  Pure host plumbing: no effect on results.
"""
from __future__ import annotations

import contextlib
import os
import subprocess
from typing import Optional, Set

import torch


def _parse_cpulist(text: str) -> Set[int]:
    cpus: Set[int] = set()
    for part in text.strip().split(','):
        if '-' in part:
            a, b = part.split('-')
            cpus.update(range(int(a), int(b) + 1))
        elif part:
            cpus.add(int(part))
    return cpus


def gpu_local_cpus(device_index: int = 0) -> Optional[Set[int]]:
    """CPUs of the NUMA node the GPU's PCIe root port hangs off, or None when the topology cannot be read."""
    bdf = None
    try:
        pr = torch.cuda.get_device_properties(device_index)
        if all(hasattr(pr, a) for a in ('pci_domain_id', 'pci_bus_id', 'pci_device_id')):
            bdf = '%04x:%02x:%02x.0' % (int(pr.pci_domain_id), int(pr.pci_bus_id), int(pr.pci_device_id))
    except Exception:
        bdf = None
    if not bdf:
        try:
            bdf = subprocess.run(['nvidia-smi', '-i', str(device_index), '--query-gpu=pci.bus_id',
                                  '--format=csv,noheader'], capture_output=True, text=True, timeout=10).stdout.strip()
        except Exception:
            return None
    if not bdf:
        return None
    bdf = bdf.lower()
    if len(bdf.split(':')[0]) == 8:        # nvidia-smi prints an 8-digit PCI domain, sysfs uses 4
        bdf = bdf[4:]
    try:
        cpus = _parse_cpulist(open('/sys/bus/pci/devices/%s/local_cpulist' % bdf).read())
    except Exception:
        return None
    cpus &= os.sched_getaffinity(0)
    return cpus or None


@contextlib.contextmanager
def gpu_local_affinity(device_index: int = 0, single_thread: bool = True):
    """Run the body on the GPU's NUMA node (and, by default, with torch's intra-op pool reduced to one thread, so
    that buffers touched inside are touched from that node only)."""
    old_aff = os.sched_getaffinity(0)
    old_threads = torch.get_num_threads()
    cpus = gpu_local_cpus(device_index)
    try:
        if cpus:
            os.sched_setaffinity(0, cpus)
        if single_thread:
            torch.set_num_threads(1)
        yield cpus
    finally:
        torch.set_num_threads(old_threads)
        os.sched_setaffinity(0, old_aff)


def pinned_like(src: torch.Tensor, device_index: int = 0) -> torch.Tensor:
    """Pinned host copy of ``src`` allocated and written from the GPU's NUMA node."""
    with gpu_local_affinity(device_index):
        out = torch.empty(src.shape, dtype=src.dtype, pin_memory=True)
        out.copy_(src)
    return out
