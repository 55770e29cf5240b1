"""Static ground-truth maps of a sequence on the GPU — the map lidiff/map_from_scans.py writes to `<seq>/map_clean.npy`.

The reference appends each filtered, transformed scan to the map and de-duplicates the whole map again (per voxel, the first point in
map order stays).  A map point is never evicted by a later scan, so that is one global first-occurrence de-duplication over all
scans in scan order; MapBuilder builds it scan by scan with a persistent GPU table of voxel keys (lb2_map_scan), O(points read).

    mb = MapBuilder(voxel_size=0.1)
    for pose, scan, labels in ...:
        mb.add_scan(scan, labels, pose)
    np.save("map_clean.npy", mb.points().cpu().numpy())

There is no CPU fallback: the builder raises without the CUDA library or an sm_90 device.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

MAX_SCAN_POINTS = 1 << 22          # points per lb2_map_scan call; larger scans are split (the first occurrence is the same either way)


def _pow2_at_least(n: int) -> int:
    return 1 << max(4, (max(int(n), 1) - 1).bit_length())


class MapBuilder:
    """voxel_size / div_mode as the reference's run: div_mode 0 divides by the voxel size (its --cpu run), 1 multiplies by the fp32
    reciprocal (PyTorch's CUDA division, its default).  initial_capacity = map rows to allocate for; table and map grow by doubling."""

    def __init__(self, voxel_size: float = 0.1, div_mode: int = 1, device="cuda", initial_capacity: int = 1 << 20):
        if not voxel_size > 0:
            raise ValueError(f"voxel_size must be > 0, got {voxel_size}")
        if div_mode not in (0, 1):
            raise ValueError(f"div_mode must be 0 or 1, got {div_mode}")
        self.h = _lib.get_handle(device)
        self.device = self.h.device
        self.voxel_size, self.div_mode = float(voxel_size), int(div_mode)
        self.n = 0
        self.rehashes = 0
        cap = max(int(initial_capacity), 1)
        self._table = self.h.new_map_table(_pow2_at_least(2 * cap))
        self.h.map_rehash(None, self._table)
        self._map = torch.empty((cap, 3), dtype=torch.float32, device=self.device)
        self._out = torch.zeros(2, dtype=torch.int32, device=self.device)
        self._scratch, self._scratch_n = None, 0
        self._failed = None

    @property
    def table_capacity(self) -> int:
        return self._table[2]

    def _reserve(self, k: int) -> None:
        """room for k more rows in the table (load <= 1/2) and in the map buffer, by doubling"""
        need = self.n + k
        cap = self._table[2]
        if cap < 2 * need:
            while cap < 2 * need:
                cap *= 2
            table = self.h.new_map_table(cap)
            self.h.map_rehash(self._table, table)
            self._table = table
            self.rehashes += 1
        rows = self._map.shape[0]
        if rows < need:
            while rows < need:
                rows *= 2
            grown = torch.empty((rows, 3), dtype=torch.float32, device=self.device)
            grown[: self.n] = self._map[: self.n]
            self._map = grown
        if self._scratch_n < k:
            self._scratch_n = _pow2_at_least(k)
            self._scratch = self.h.map_scan_scratch(self._scratch_n)

    def _as_points(self, points) -> torch.Tensor:
        t = torch.as_tensor(points)
        if t.dim() != 2 or t.shape[1] != 4 or t.dtype != torch.float32:
            raise ValueError(f"points must be a float32 (n, 4) array of x, y, z, remission rows, got {tuple(t.shape)} {t.dtype}")
        return t.to(self.device, non_blocking=True).contiguous()

    def _as_labels(self, labels, n: int):
        if labels is None:
            return None
        if isinstance(labels, np.ndarray):
            if labels.dtype not in (np.uint32, np.int32):
                raise ValueError(f"labels must be uint32 (or int32), got {labels.dtype}")
            labels = torch.from_numpy(labels.view(np.int32))
        elif labels.dtype == torch.uint32:
            labels = labels.view(torch.int32)
        if labels.dtype != torch.int32 or labels.dim() != 1 or labels.shape[0] != n:
            raise ValueError(f"labels must be {n} 32-bit values, got {tuple(labels.shape)} {labels.dtype}")
        return labels.to(self.device, non_blocking=True).contiguous()

    @staticmethod
    def _pose12(pose) -> list:
        """the first three rows of the 4x4 pose, rounded to fp32 as the reference's `.float()` does"""
        if pose is None:
            return [1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0]
        p = np.asarray(pose, dtype=np.float64)
        if p.shape not in ((4, 4), (3, 4)):
            raise ValueError(f"pose must be 4x4 or 3x4, got {p.shape}")
        return [float(v) for v in p[:3, :4].astype(np.float32).reshape(-1)]

    def add_scan(self, points_xyzr, labels=None, pose=None) -> int:
        """filters (labels: class (l & 0xFFFF) in (1, 252); range: |(x, y, z, remission)| > 3.5), transforms by `pose` (4x4, the scan
        to the map frame; None = identity) and adds the points of new voxels.  Returns the number of rows added."""
        if self._failed:
            raise RuntimeError(f"MapBuilder: an earlier scan failed ({self._failed}); the map is incomplete")
        pts = self._as_points(points_xyzr)
        lab = self._as_labels(labels, pts.shape[0])
        pose12 = self._pose12(pose)
        added = 0
        for s in range(0, pts.shape[0], MAX_SCAN_POINTS):
            e = min(pts.shape[0], s + MAX_SCAN_POINTS)
            self._reserve(e - s)
            self.h.map_scan(pts[s:e], lab[s:e] if lab is not None else None, pose12, self.voxel_size, self.div_mode, self._table,
                            self._map, self.n, self._out, self._scratch)
            new, status = (int(v) for v in self._out.tolist())          # the one host read per call: the row count and the status
            if status:
                self._failed = "a voxel index outside +-2^20 voxels per axis"
                raise ValueError(f"MapBuilder: a point of the scan lies outside the map's key range (+-{2 ** 20} voxels of "
                                 f"{self.voxel_size} m per axis)")
            self.n += new
            added += new
        return added

    def points(self) -> torch.Tensor:
        """(M, 3) float32 map rows in first-occurrence order (a view of the builder's buffer, valid until the next add_scan)"""
        return self._map[: self.n]
