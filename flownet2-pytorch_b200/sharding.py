"""Data-parallel sharding helpers -- the H100-native stand-in for the reference's
``nn.DataParallel`` wrapper (main.py:189,200: effective batch = batch_size x number_gpus).

One process per GPU (``torchrun``); the three layers and the whole FlowNet2 forward are per-sample,
so the batch dimension is split evenly and NO collective sits on the data path.  ``torch.distributed``
(NCCL over NVLink on the box, gloo in the CPU tests) is used only for barriers, the max-over-ranks
timing reduction and an optional gather of the output flows.
"""
import torch
import torch.distributed as dist


def shard_range(n, world, rank):
    """Contiguous [lo, hi) slice of ``n`` samples owned by ``rank``; the first ``n % world`` ranks get
    one extra sample (same split torch's scatter uses)."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad world/rank %d/%d" % (world, rank))
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(t, world=None, rank=None, dim=0):
    world = dist.get_world_size() if world is None else world
    rank = dist.get_rank() if rank is None else rank
    lo, hi = shard_range(t.size(dim), world, rank)
    return t.narrow(dim, lo, hi - lo)


def gather_batch(local, total, dim=0):
    """All-gather per-rank shards of possibly unequal size back into the full batch (every rank gets it)."""
    world, rank = dist.get_world_size(), dist.get_rank()
    sizes = [shard_range(total, world, r) for r in range(world)]
    maxn = max(hi - lo for lo, hi in sizes)
    pad_shape = list(local.shape)
    pad_shape[dim] = maxn
    buf = local.new_zeros(pad_shape)
    buf.narrow(dim, 0, local.size(dim)).copy_(local)
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf)
    return torch.cat([p.narrow(dim, 0, hi - lo) for p, (lo, hi) in zip(parts, sizes)], dim=dim)


def max_over_ranks(value, device=None):
    """Timing reduction used by bench.py: a job is as slow as its slowest rank."""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])
