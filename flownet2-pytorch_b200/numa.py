"""NUMA placement of a rank's host staging buffers (one process per GPU).

Pinned host memory is allocated on the NUMA node of the thread that calls ``cudaHostAlloc`` (first touch
under that thread's CPU affinity / memory policy).  ``torchrun`` starts every rank without any affinity, so
on a two-socket box half of the ranks stage their H2D / D2H traffic through the remote socket's memory
controller and the inter-socket link, which slows the host-buffer (``e2e``) step as ranks are added while the
kernels scale perfectly.

``bind_to_device_node(dev)`` pins the calling process (CPU affinity + ``set_mempolicy(MPOL_PREFERRED)``)
to the NUMA node the GPU's PCIe root port hangs off.  Call it BEFORE allocating pinned buffers.
Everything here is Linux sysfs + two syscalls; it imports neither torch's CUDA state nor libfn2b200
(bench.py loads it by path for the reference arm too).  Failure is never fatal: the function returns a
dict that says what it did (``{"node": None, ...}`` when the topology cannot be read).
"""
import ctypes
import os

_SYS_NODE = "/sys/devices/system/node"
MPOL_DEFAULT, MPOL_PREFERRED, MPOL_BIND = 0, 1, 2
_NR_SET_MEMPOLICY = 238          # x86_64


def parse_cpulist(text):
    """'0-3,8,10-11' -> [0,1,2,3,8,10,11] (the format of /sys/devices/system/node/nodeN/cpulist)."""
    cpus = []
    for part in text.strip().split(","):
        part = part.strip()
        if not part:
            continue
        if "-" in part:
            lo, hi = part.split("-", 1)
            cpus.extend(range(int(lo), int(hi) + 1))
        else:
            cpus.append(int(part))
    return cpus


def pci_address(domain, bus, device, function=0):
    """sysfs name of a PCI function, e.g. (0, 0x1b, 0) -> '0000:1b:00.0'."""
    return "%04x:%02x:%02x.%d" % (domain, bus, device, function)


def node_of_pci(addr, sysfs="/sys/bus/pci/devices"):
    """NUMA node of a PCI device (-1 / missing file -> None)."""
    try:
        n = int(open(os.path.join(sysfs, addr, "numa_node")).read().strip())
    except (OSError, ValueError):
        return None
    return n if n >= 0 else None


def node_cpus(node, sysnode=_SYS_NODE):
    try:
        return parse_cpulist(open(os.path.join(sysnode, "node%d" % node, "cpulist")).read())
    except (OSError, ValueError):
        return []


def online_nodes(sysnode=_SYS_NODE):
    try:
        return sorted(int(d[4:]) for d in os.listdir(sysnode) if d.startswith("node") and d[4:].isdigit())
    except OSError:
        return []


def device_node(device_index):
    """NUMA node of CUDA device `device_index` (through torch's device properties), or None."""
    import torch
    p = torch.cuda.get_device_properties(device_index)
    return node_of_pci(pci_address(p.pci_domain_id, p.pci_bus_id, p.pci_device_id))


def set_preferred_node(node):
    """set_mempolicy(MPOL_PREFERRED, {node}) for the calling thread; returns True on success.  PREFERRED (not BIND):
    an exhausted node falls back to the other one instead of failing the allocation."""
    try:
        libc = ctypes.CDLL(None, use_errno=True)
        nbits = max(64, ((max(online_nodes() or [node]) + 1 + 63) // 64) * 64)
        mask = (ctypes.c_ulong * (nbits // 64))()
        mask[node // 64] |= 1 << (node % 64)
        rc = libc.syscall(_NR_SET_MEMPOLICY, ctypes.c_int(MPOL_PREFERRED), ctypes.byref(mask), ctypes.c_ulong(nbits + 1))
        return rc == 0
    except Exception:
        return False


def bind_to_node(node):
    """CPU affinity + preferred memory node for this process.  Returns what was done."""
    info = {"node": node, "cpus": 0, "affinity": False, "mempolicy": False}
    if node is None:
        return info
    cpus = node_cpus(node)
    allowed = set(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else set()
    use = sorted(set(cpus) & allowed) if allowed else cpus
    if use:
        try:
            os.sched_setaffinity(0, use)
            info["affinity"], info["cpus"] = True, len(use)
        except OSError:
            pass
    info["mempolicy"] = set_preferred_node(node)
    return info


def bind_to_device_node(device_index):
    """Bind this process to the NUMA node of CUDA device `device_index`; call before allocating pinned buffers."""
    if os.environ.get("FN2B200_NUMA", "1") == "0":
        return {"node": None, "cpus": 0, "affinity": False, "mempolicy": False, "disabled": True}
    try:
        node = device_node(device_index)
    except Exception:
        node = None
    return bind_to_node(node)
