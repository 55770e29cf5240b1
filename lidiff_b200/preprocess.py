"""`preprocess_scan` pieces on the GPU (/root/reference/lidiff/tools/diff_completion_pipeline.py:92-105).

`farthest_point_sample` replaces open3d's `PointCloud.farthest_point_down_sample` (start at point 0,
repeatedly take the first argmax of the running min squared distance, fp64) and, like open3d's
`SelectByIndex`, returns the selection in ORIGINAL index order.
"""
from __future__ import annotations

import torch

from . import _lib


def farthest_point_sample(points: torch.Tensor, n_samples: int, ordered: bool = True) -> torch.Tensor:
    if not points.is_cuda:
        raise RuntimeError("farthest_point_sample: CUDA tensor required (no CPU fallback)")
    pts = points.to(torch.float64).contiguous()
    n = pts.shape[0]
    if n_samples > n:
        raise RuntimeError(f"farthest_point_sample: asked for {n_samples} of {n} points")
    h = _lib.get_handle(pts.device)
    idx = torch.empty(n_samples, dtype=torch.int32, device=pts.device)
    dist = torch.empty(n, dtype=torch.float64, device=pts.device)
    h.farthest_point_sample(pts, n, n_samples, idx, dist)
    idx = idx.long()
    return torch.sort(idx).values if ordered else idx


def farthest_point_sample_batched(scans: list[torch.Tensor], n_samples: int, ordered: bool = True) -> torch.Tensor:
    """`farthest_point_sample` of every scan of `scans` (CUDA (n_b, 3) tensors of any sizes >= n_samples) in one launch of the
    cluster kernel: (B, n_samples) int64 scan-local indices, each row equal to farthest_point_sample(scans[b], n_samples).
    Scans larger than the kernel's on-chip capacity are sampled one by one with the single-scan kernel."""
    if not all(s.is_cuda for s in scans):
        raise RuntimeError("farthest_point_sample_batched: CUDA tensors required (no CPU fallback)")
    sizes = [int(s.shape[0]) for s in scans]
    if not scans or min(sizes) < n_samples:
        raise RuntimeError(f"farthest_point_sample_batched: asked for {n_samples} of {min(sizes, default=0)} points")
    dev = scans[0].device
    h = _lib.get_handle(dev)
    out = torch.empty((len(scans), n_samples), dtype=torch.int64, device=dev)
    cap = h.fps_batched_capacity()
    on_chip = [b for b, n in enumerate(sizes) if n <= cap]
    for b in range(len(scans)):
        if b not in on_chip:
            out[b] = farthest_point_sample(scans[b], n_samples, ordered=False)
    if on_chip:
        pts = torch.cat([scans[b].to(torch.float64).reshape(-1, 3) for b in on_chip]).contiguous()
        offsets = torch.tensor([0] + [sizes[b] for b in on_chip], dtype=torch.int64).cumsum(0).to(dev)
        idx = torch.empty((len(on_chip), n_samples), dtype=torch.int32, device=dev)
        h.farthest_point_sample_batched(pts, offsets, len(on_chip), max(sizes[b] for b in on_chip), n_samples, idx)
        out[on_chip] = idx.long()
    return torch.sort(out, dim=1).values if ordered else out
