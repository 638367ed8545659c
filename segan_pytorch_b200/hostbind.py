"""Host-side placement for the pinned staging buffers (train.py / clean.py / bench.py).

A pinned buffer lands on the NUMA node of the thread that first touches it.  On a two-socket GPU host a process
started on the far socket stages every batch across the inter-socket link, and the one-step-ahead upload of
DevicePrefetcher may then no longer hide behind the step.  `bind_host_to_gpu` restricts the calling process to the CPUs that sysfs reports as local to the
GPU's PCIe root *before* those buffers are allocated; it never widens the affinity it was given and does nothing when
the information is missing."""
import os

import torch


def parse_cpulist(text):
    """'0-3,8,10-11' -> {0, 1, 2, 3, 8, 10, 11} (the sysfs cpulist format)."""
    cpus = set()
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.update(range(int(lo), int(hi or lo) + 1))
    return cpus


def gpu_local_cpus(device):
    """CPUs local to `device` (sysfs local_cpulist of its PCI function), or None."""
    try:
        props = torch.cuda.get_device_properties(device)
        addr = "%04x:%02x:%02x.0" % (props.pci_domain_id, props.pci_bus_id, props.pci_device_id)
        with open("/sys/bus/pci/devices/%s/local_cpulist" % addr) as f:
            text = f.read().strip()
    except Exception:
        return None
    return parse_cpulist(text) or None


def bind_host_to_gpu(device):
    """Returns the CPU set the process now runs on (or None when nothing was changed)."""
    if os.environ.get("SEGAN_B200_NUMA_BIND", "1").lower() in ("0", "off", "no", "false"):
        return None
    if not hasattr(os, "sched_getaffinity"):
        return None
    local = gpu_local_cpus(device)
    if not local:
        return None
    try:
        mine = os.sched_getaffinity(0)
        want = mine & local
        if not want or want == mine:
            return None
        os.sched_setaffinity(0, want)
        return want
    except OSError:
        return None
