"""Data-parallel training under torchrun, as the reference's training scripts run Lightning's `accelerator='ddp'` on every GPU present
(lidiff/train.py:88-101, lidiff/train_refine.py:56-70): one process per rank, synchronised batch norm (me.MinkowskiSyncBatchNorm),
DistributedDataParallel averaging the gradients, and each rank's own shard of the data (DistributedSampler).

Without torchrun's environment (WORLD_SIZE unset or 1) nothing here is used and the training CLIs run as one process."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist
from torch.utils.data import DataLoader, DistributedSampler


class Run:
    """this process' place in the run: rank, world size and device (world 1: a single-process run, no process group)"""

    def __init__(self, rank=0, world=1, device=None):
        self.rank, self.world = rank, world
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())

    @property
    def distributed(self) -> bool:
        return self.world > 1

    @property
    def main(self) -> bool:
        return self.rank == 0


def start() -> Run:
    """join torchrun's process group when WORLD_SIZE > 1.  The backend follows from what the process can observe: NCCL when every
    local rank has a device of its own (cuda:LOCAL_RANK), gloo when ranks share devices (e.g. several ranks on one GPU)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return Run()
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    local_world = int(os.environ.get("LOCAL_WORLD_SIZE", str(world)))
    ndev = torch.cuda.device_count()
    own = ndev >= local_world
    device = torch.device("cuda", local_rank if own else local_rank % max(ndev, 1))
    torch.cuda.set_device(device)
    dist.init_process_group("nccl" if own else "gloo", device_id=device if own else None)
    return Run(dist.get_rank(), dist.get_world_size(), device)


def finish(run: Run):
    if run.distributed:
        dist.barrier()
        dist.destroy_process_group()


def wrap(module, run: Run):
    """(the module to call, the module whose state_dict is saved): sync batch norm and DistributedDataParallel when distributed.
    broadcast_buffers=False: the synchronised batch norm keeps the running statistics equal on every rank."""
    if not run.distributed:
        return module, module
    from . import me as ME
    module = ME.MinkowskiSyncBatchNorm.convert_sync_batchnorm(module)
    return torch.nn.parallel.DistributedDataParallel(module, broadcast_buffers=False), module


def sharded(loader: DataLoader, run: Run, shuffle: bool) -> DataLoader:
    """the same loader over this rank's shard: DistributedSampler(shuffle, seed 0, no drop_last), which pads the shards to equal length
    so that every rank runs the same number of batches.  Single process: the loader itself."""
    if not run.distributed:
        return loader
    sampler = DistributedSampler(loader.dataset, num_replicas=run.world, rank=run.rank, shuffle=shuffle, seed=0, drop_last=False)
    return DataLoader(loader.dataset, batch_size=loader.batch_size, sampler=sampler, num_workers=0, collate_fn=loader.collate_fn)


def set_epoch(loader: DataLoader, epoch: int):
    if isinstance(loader.sampler, DistributedSampler):
        loader.sampler.set_epoch(epoch)


def mean_over_ranks(values, run: Run, device) -> list[float]:
    """the mean over ranks of a list of scalars (one all-reduce); single process: the values"""
    if not run.distributed:
        return [float(v) for v in values]
    t = torch.tensor([float(v) for v in values], dtype=torch.float64, device=device)
    dist.all_reduce(t)
    t /= run.world
    return t.tolist()
