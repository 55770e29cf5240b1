"""Builds the static ground-truth map of each sequence — counterpart of the reference's `python lidiff/map_from_scans.py -p PATH
[-v 0.1]` (lidiff/map_from_scans.py:55-96): for every sequence 00..10 under PATH, the scans velodyne/*.bin (natural order, zipped with
poses.txt, so the shorter list wins) without moving classes and flying artefacts, in the map frame (poses.txt through calib.txt's
Tr when it exists), de-duplicated on a voxel grid; written to PATH/<seq>/map_clean.npy as float32 (M, 3), first occurrence first.

    python -m lidiff_b200.tools.map_from_scans -p ./Datasets/SemanticKITTI/dataset/sequences
    torchrun --nproc-per-node 8 -m lidiff_b200.tools.map_from_scans -p ... --sequences 00 --sequences 08

The map is built on the GPU (lidiff_b200.maps.MapBuilder) in one pass over the scans; a reader thread loads the next scan's .bin and
.label into pinned host buffers while the GPU inserts the current one.  --div-mode 1 (default) divides by the voxel size as PyTorch
does on the GPU (the reference's default device), 0 as it does on the CPU.  Under torchrun sequence i runs on rank i mod R.
"""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor

import click
import numpy as np
import torch

from ..kitti import label_path, load_poses, natural_sorted, read_labels, read_scan
from ..maps import MapBuilder
from ..sharding import scans_of_rank

SEQUENCES = ["00", "01", "02", "03", "04", "05", "06", "07", "08", "09", "10"]


def sequence_scans(seq_dir: str) -> list:
    """[(4x4 LiDAR-frame pose, scan path)] as the reference pairs them: zip(poses, natsorted(velodyne/)), truncated to the shorter"""
    poses = load_poses(os.path.join(seq_dir, "calib.txt"), os.path.join(seq_dir, "poses.txt"))
    names = natural_sorted(os.listdir(os.path.join(seq_dir, "velodyne")))
    return [(pose, os.path.join(seq_dir, "velodyne", name)) for pose, name in zip(poses, names)]


class ScanReader:
    """reads (points, labels) of a scan into one of two alternating host buffers (pinned when a GPU is present); the caller reads
    scan k + 1 into the other buffer while scan k is in use, and must be done with a buffer before it is read into again"""

    def __init__(self, pin: bool):
        self.pin = pin
        self._bufs = [[None, None], [None, None]]

    def _buffer(self, slot: int, j: int, nbytes: int) -> torch.Tensor:
        b = self._bufs[slot][j]
        if b is None or b.numel() < nbytes:
            b = torch.empty(max(nbytes + nbytes // 4, 1 << 16), dtype=torch.uint8, pin_memory=self.pin)
            self._bufs[slot][j] = b
        return b

    def read(self, slot: int, scan_path: str, with_labels: bool = True):
        buf = self._buffer(slot, 0, os.path.getsize(scan_path))
        n = read_scan(scan_path, out=buf.numpy()).shape[0]
        points = buf[: 16 * n].view(torch.float32).view(n, 4)
        if not with_labels:
            return points, None
        lpath = label_path(scan_path)
        lbuf = self._buffer(slot, 1, os.path.getsize(lpath) if os.path.exists(lpath) else 0)     # read_labels names a missing file
        read_labels(lpath, n, out=lbuf.numpy())
        return points, lbuf[: 4 * n].view(torch.int32)


def build_sequence_map(seq_dir: str, voxel_size: float = 0.1, div_mode: int = 1, device="cuda", reader: ScanReader | None = None,
                       with_labels: bool = True) -> np.ndarray:
    """the map of one sequence as a float32 (M, 3) array"""
    scans = sequence_scans(seq_dir)
    mb = MapBuilder(voxel_size, div_mode, device)
    reader = reader or ScanReader(pin=mb.device.type == "cuda")
    with ThreadPoolExecutor(max_workers=1) as pool:
        pending = pool.submit(reader.read, 0, scans[0][1], with_labels) if scans else None
        for k, (pose, _) in enumerate(scans):
            points, labels = pending.result()
            if k + 1 < len(scans):                       # the other buffer: add_scan below has finished with it (it synchronises)
                pending = pool.submit(reader.read, (k + 1) % 2, scans[k + 1][1], with_labels)
            mb.add_scan(points, labels, pose)
    return mb.points().cpu().numpy()


def parse_sequences(values) -> list:
    """--sequences 00 --sequences 08, or --sequences 00,08"""
    if not values:
        return list(SEQUENCES)
    return [s.strip() for v in values for s in v.split(",") if s.strip()]


@click.command()
@click.option("--path", "-p", type=str, required=True, help="path to the scan sequences (the directory holding 00, 01, ...)")
@click.option("--voxel_size", "-v", type=float, default=0.1, help="voxel size")
@click.option("--cpu", "-c", is_flag=True, help="Use CPU (not supported: the map is built on the GPU)")
@click.option("--sequences", multiple=True, help="sequences to build (repeatable or comma-separated; default 00..10)")
@click.option("--div-mode", type=click.IntRange(0, 1), default=1,
              help="voxel index arithmetic: 1 = x * fp32(1 / voxel_size) (PyTorch on the GPU), 0 = x / voxel_size (PyTorch on the CPU)")
def main(path, voxel_size, cpu, sequences, div_mode):
    if cpu:
        raise click.UsageError("there is no CPU path: maps are built on the GPU (use --div-mode 0 for the reference's --cpu arithmetic)")
    seqs = parse_sequences(sequences)
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    if torch.cuda.is_available():
        torch.cuda.set_device(device)
    if world > 1:                        # the only collective is the final barrier: gloo, no device communicator
        import torch.distributed as dist
        dist.init_process_group("gloo")
    try:
        for i in scans_of_rank(len(seqs), world, rank):
            seq = seqs[i]
            points = build_sequence_map(os.path.join(path, seq), voxel_size, div_mode, device)
            print(f"saving map for sequence {seq}")
            np.save(os.path.join(path, seq, "map_clean.npy"), points)
    finally:
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
