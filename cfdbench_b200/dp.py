"""Data-parallel plumbing for the FNO path (one process per GPU, torch.distributed).

The reference has no distributed code at all (SURVEY.md 2, 8e).  Rollout shards the batch of cases
with no collective; training needs exactly one exchange per step: the mean of one flat float32
gradient buffer (2,368,354 reals for cavity), all-reduced over NCCL (gloo in CPU tests).
"""
from __future__ import annotations

import os
from typing import Tuple

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None) -> Tuple[int, int, int]:
    """Initialise torch.distributed from torchrun's env (RANK/LOCAL_RANK/WORLD_SIZE/MASTER_*).
    Returns (rank, local_rank, world_size); a no-op single-process setup when WORLD_SIZE is unset."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, local, world


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [begin, end) slice of `total` cases owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(total, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def allreduce_mean_(flat: torch.Tensor, group=None) -> torch.Tensor:
    """In-place mean over the group of a flat real gradient buffer (complex parameters are exposed as
    interleaved reals so the collective never sees a complex dtype)."""
    if flat.is_complex():
        raise TypeError("pass the real view of complex gradients")
    if dist.get_backend(group) == "nccl":   # averaged inside the collective: no separate division kernel
        dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=group)
    else:                                    # gloo (CPU tests) has no AVG
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.div_(dist.get_world_size(group))
    return flat


def max_over_ranks(value: float, device=None) -> float:
    """Max of a host scalar over all ranks (used for the bench's max-over-ranks timing)."""
    if not dist.is_initialized():
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
