"""B x H sharding of the FFT-convolution path across the GPUs of one box.

Every (b, h) convolution is independent and dk[h] is a sum over b only, so sharding the CHANNEL axis needs no
collective in forward or backward: each rank owns a contiguous block of channels of u, k (and gates) and
produces the same block of y / du / dk.  The only communication is harness-side: gathering the blocks for a
parity check (torch.distributed all_gather over NCCL / NVLink on GPUs, gloo in the CPU tests).
"""
import os

import torch
import torch.distributed as dist


def channel_range(H, world, rank):
    """Contiguous channel block [h0, h1) of `rank`; blocks differ by at most one channel."""
    base, rem = divmod(H, world)
    h0 = rank * base + min(rank, rem)
    return h0, h0 + base + (1 if rank < rem else 0)


def shard(u, k, world, rank, *gates):
    """Slices of (B,H,L) tensors and the (H,Lk) filter owned by `rank` (contiguous copies).  A grouped filter (G < H
    rows shared by groups of channels) is refused: a channel block can split a group."""
    if k.dim() != 2 or k.shape[0] != u.shape[1]:
        raise RuntimeError(f'shard: k must be (H={u.shape[1]}, Lk), got {tuple(k.shape)}; grouped filters are not '
                           'sharded')
    h0, h1 = channel_range(u.shape[1], world, rank)
    out = [u[:, h0:h1].contiguous(), k[h0:h1].contiguous()]
    out += [g[:, h0:h1].contiguous() for g in gates]
    return out


def gather_channels(y_local, H, group=None):
    """All-gather channel blocks (B, Hr, L) -> (B, H, L) on every rank (harness only, not on the hot path)."""
    world = dist.get_world_size(group)
    B, _, L = y_local.shape
    hmax = (H + world - 1) // world
    pad = torch.zeros((B, hmax, L), dtype=y_local.dtype, device=y_local.device)
    pad[:, : y_local.shape[1]] = y_local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    parts = []
    for r in range(world):
        h0, h1 = channel_range(H, world, r)
        parts.append(bufs[r][:, : h1 - h0])
    return torch.cat(parts, dim=1)


def sharded_conv(conv_fn, u, k, group=None, gates=()):
    """Run `conv_fn(u_r, k_r, *gates_r)` on this rank's channel block and gather the full output."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    parts = shard(u, k, world, rank, *gates)
    y_local = conv_fn(*parts)
    return gather_channels(y_local, u.shape[1], group)


def _cpulist(text):
    cpus = set()
    for part in text.strip().split(','):
        if '-' in part:
            a, b = part.split('-')
            cpus.update(range(int(a), int(b) + 1))
        elif part:
            cpus.add(int(part))
    return cpus


def bind_to_gpu_numa_node(device_index):
    """Bind this process's CPU affinity to the cores of the NUMA node the GPU hangs off (sysfs: the PCI device's
    `numa_node`, then /sys/devices/system/node/nodeN/cpulist).  Host staging buffers allocated and first touched after
    this call (pinned memory for forward_host) then live on that node, so H2D / D2H copies of the ranks of one box do
    not all cross the inter-socket link.  One process per GPU (torchrun) is the assumed launch.  Returns a description."""
    import torch.cuda
    bus = torch.cuda.get_device_properties(device_index)
    pci = f'{bus.pci_domain_id:04x}:{bus.pci_bus_id:02x}:{bus.pci_device_id:02x}.0'
    node = int(open(f'/sys/bus/pci/devices/{pci}/numa_node').read())
    if node < 0:
        return f'gpu {device_index} ({pci}): no NUMA affinity reported'
    cpus = _cpulist(open(f'/sys/devices/system/node/node{node}/cpulist').read())
    allowed = os.sched_getaffinity(0) & cpus
    if not allowed:
        return f'gpu {device_index} ({pci}): node {node} has no allowed cpus'
    os.sched_setaffinity(0, allowed)
    try:            # prefer the node for new pages too (a no-op where set_mempolicy is not permitted)
        import ctypes
        libc = ctypes.CDLL(None, use_errno=True)
        mask = ctypes.c_ulong(1 << node)
        libc.syscall(238, 1, ctypes.byref(mask), ctypes.c_ulong(64))      # set_mempolicy(MPOL_PREFERRED) on x86-64
    except Exception:
        pass
    return f'gpu {device_index} ({pci}): bound to NUMA node {node}, {len(allowed)} cpus'
