"""Batch-dimension sharding of whole scans across ranks (SURVEY.md 8e).

The per-scan sparse graph does not partition, so multi-GPU = one process per GPU, scan b on rank
b mod R, no collective in the data path.  torch.distributed (NCCL on GPUs, gloo in the CPU tests) is
used only to (1) bracket the timed region with barriers, (2) reduce the per-rank device time with MAX and
(3) gather the variable-length per-scan results at the end.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def scans_of_rank(n_scans: int, world: int, rank: int) -> list[int]:
    """scan b runs on rank b mod world"""
    return [b for b in range(n_scans) if b % world == rank]


def batches_of_rank(n_scans: int, world: int, rank: int, batch: int) -> list[list[int]]:
    """the scans of this rank (scans_of_rank) in groups of `batch`, in order; the last group may be shorter"""
    if batch < 1:
        raise ValueError(f"batch size must be >= 1, got {batch}")
    mine = scans_of_rank(n_scans, world, rank)
    return [mine[i:i + batch] for i in range(0, len(mine), batch)]


def max_over_ranks(ms: float, device) -> float:
    """the job's time is the slowest rank's device time"""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(ms)
    t = torch.tensor([ms], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_scans(local: dict[int, torch.Tensor], n_scans: int, device) -> dict[int, torch.Tensor] | None:
    """all ranks -> rank 0: {scan index: (n_i, 3) completed points}.  Variable lengths are exchanged first,
    then one padded all_gather (NCCL/gloo have no variable-size gather)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return dict(local)
    world, rank = dist.get_world_size(), dist.get_rank()
    lens = torch.zeros(n_scans, dtype=torch.int64, device=device)
    for b, pts in local.items():
        lens[b] = pts.shape[0]
    dist.all_reduce(lens, op=dist.ReduceOp.SUM)
    per_rank = max(len(scans_of_rank(n_scans, world, r)) for r in range(world))
    width = int(lens.max().item())
    buf = torch.zeros((per_rank, width, 3), dtype=torch.float32, device=device)
    for slot, b in enumerate(scans_of_rank(n_scans, world, rank)):
        buf[slot, : local[b].shape[0]] = local[b].to(device=device, dtype=torch.float32)
    out = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(out, buf)
    if rank != 0:
        return None
    res = {}
    for r in range(world):
        for slot, b in enumerate(scans_of_rank(n_scans, world, r)):
            res[b] = out[r][slot, : int(lens[b].item())]
    return res
