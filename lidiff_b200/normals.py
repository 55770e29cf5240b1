"""Point normals on the GPU — the counterpart of open3d 0.17's `PointCloud.estimate_normals()`, which the reference's inference
script calls on the refined and the diffusion cloud of every scan before writing them (tools/diff_completion_pipeline.py:204-212):

  * `knn(points, k)`: exact self-k-nearest neighbours (k <= 32) over the Morton-sorted box tree of lidiff_b200.metrics
    (lb2_pc_tree_build / lb2_pc_knn), the point itself included, ordered by (d², index) — ties go to the lower index;
  * `estimate_normals(points, knn=30)`: open3d's one-pass cumulant covariance of those neighbours and its FastEigen3x3 eigensolver
    (lb2_pc_normals), unoriented, (0, 0, 1) where the solver gives the zero vector.

Points may be numpy arrays, torch tensors on any device, or open3d-shim PointClouds.  There is no CPU fallback."""
from __future__ import annotations

import torch

from . import _lib
from .metrics import _points

MAX_K = 32


def _check_k(k) -> int:
    k = int(k)
    if not 1 <= k <= MAX_K:
        raise ValueError(f"k-nearest neighbours: k must be in [1, {MAX_K}], got {k}")
    return k


def knn(points, k: int, device="cuda"):
    """(idx int32 (n, min(k, n)), d2 fp64 (n, min(k, n))) device tensors: row j lists the points nearest to point j in (squared
    distance, index) order, itself first unless a duplicate with a lower index precedes it.  Exact for finite coordinates; a slot
    the search cannot fill holds index -1 and d2 = +inf (every slot of a point with a NaN or infinite coordinate, and the slots
    past the number of finite points)"""
    k = _check_k(k)
    h = _lib.get_handle(device)
    p = _points(points, h.device)
    n = p.shape[0]
    ke = min(k, n)
    idx = torch.empty((n, ke), dtype=torch.int32, device=h.device)
    d2 = torch.empty((n, ke), dtype=torch.float64, device=h.device)
    if n:
        h.pc_knn(h.pc_tree(p), n, ke, idx, d2)
    return idx, d2


def estimate_normals(points, knn: int = 30, device="cuda") -> torch.Tensor:
    """(n, 3) fp64 device tensor: open3d's estimate_normals(KDTreeSearchParamKNN(knn)) of the cloud, without orientation; NaN for a
    point whose neighbour row has an empty slot (see `knn`)"""
    k = _check_k(knn)
    h = _lib.get_handle(device)
    p = _points(points, h.device)
    n = p.shape[0]
    out = torch.empty((n, 3), dtype=torch.float64, device=h.device)
    if n:
        ke = min(k, n)
        idx = torch.empty((n, ke), dtype=torch.int32, device=h.device)
        h.pc_knn(h.pc_tree(p), n, ke, idx)
        h.pc_normals(p, idx, out)
    return out
