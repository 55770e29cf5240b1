"""TEST INFRASTRUCTURE: a numpy stand-in for the refinement-sample methods of `lidiff_b200._lib.Handle` (lb2_aggregate_window,
lb2_jitter_filter, lb2_voxel_first_f64) and for pc_tree / pc_nn, on top of the CPU fake of tests/fake_backend.py, so the host logic
of lidiff_b200.datasets_refine and metrics.chamfer_distance can be exercised without a GPU.  The `restate_*` functions restate the
kernels' documented arithmetic in numpy (every operation rounded, no FMA, in the header's order) and are also the yardstick of the
GPU tests.  Tests install it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_backend
import metrics_reference
from lidiff_b200 import _lib
from lidiff_b200.datasets_refine import SEGMENT_DTYPE

KEY_HALF = 1 << 20          # voxel indices of the map keys: [-2^20, 2^20) per axis


def _rigid(m, x, y, z):
    """((m0 x + m1 y) + m2 z) + m3 per output axis; m (.., 12) broadcast against the rows"""
    m = np.asarray(m, dtype=np.float64)
    return [((m[..., 4 * k] * x + m[..., 4 * k + 1] * y) + m[..., 4 * k + 2] * z) + m[..., 4 * k + 3] for k in range(3)]


def restate_aggregate(points, labels, starts, poses, undo12, split):
    """(fp64 (m, 3) rows lb2_aggregate_window keeps in input order, rows kept of [0, split))"""
    p = np.asarray(points, dtype=np.float32).reshape(-1, 4)
    n = p.shape[0]
    lab = np.asarray(labels).view(np.uint32) & np.uint32(0xFFFF)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.sqrt((x * x + y * y) + z * z)
        keep = (lab < 252) & (d > np.float32(3.5))
        seg = np.searchsorted(np.asarray(starts, dtype=np.int64), np.arange(n), side="right") - 1
        m = np.asarray(poses, dtype=np.float64).reshape(-1, 12)[seg]
        a = _rigid(m, x.astype(np.float64), y.astype(np.float64), z.astype(np.float64))
        w = np.stack(_rigid(np.asarray(undo12, dtype=np.float64), *a), 1)
    return w[keep], int(keep[:split].sum())


def restate_jitter(points, randn, sigma, clip, max_range):
    """fp64 rows lb2_jitter_filter keeps, in input order"""
    p, r = np.asarray(points, dtype=np.float64), np.asarray(randn, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        w = np.minimum(np.maximum(sigma * r, -clip), clip) + p
        x, y, z = w[:, 0], w[:, 1], w[:, 2]
        keep = np.sqrt((x * x + y * y) + z * z) < max_range
    return w[keep]


def restate_voxel_first(points, voxel, max_range):
    """(fp64 rows lb2_voxel_first_f64 keeps in row order, status)"""
    p = np.asarray(points, dtype=np.float64)
    fin = np.isfinite(p).all(1)
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.floor(p / voxel)
    ok = fin & ((q >= -KEY_HALF) & (q < KEY_HALF)).all(1)
    status = int((fin & ~ok).any())
    rows = np.nonzero(ok)[0]
    c = q[rows].astype(np.int64) + KEY_HALF
    keys = (c[:, 0] << 42) | (c[:, 1] << 21) | c[:, 2]
    _, first = np.unique(keys, return_index=True)
    win = np.sort(rows[first])
    w = p[win]
    with np.errstate(invalid="ignore", over="ignore"):
        keep = np.sqrt((w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1]) + w[:, 2] * w[:, 2]) < max_range
    return w[keep], status


class FakeRefineHandle(fake_backend.FakeHandle):
    def _scratch(self, n):
        return torch.empty(16, dtype=torch.uint8)

    aggregate_window_scratch = jitter_filter_scratch = voxel_first_f64_scratch = _scratch

    def aggregate_window(self, points, labels, segments, nseg, undo12, split, out, d_out, scratch):
        assert points.dtype == torch.float32 and points.shape[1] == 4 and labels.shape[0] == points.shape[0]
        self.launches += 4
        seg = segments.numpy().view(SEGMENT_DTYPE)[:nseg]
        w, n_before = restate_aggregate(points.numpy(), labels.numpy(), seg["start"], seg["m"], undo12, split)
        out[: w.shape[0]] = torch.from_numpy(w)
        d_out[0], d_out[1] = w.shape[0], n_before

    def jitter_filter(self, points, randn, sigma, clip, max_range, out, d_count, scratch):
        assert points.dtype == randn.dtype == out.dtype == torch.float64
        self.launches += 3
        w = restate_jitter(points.numpy(), randn.numpy(), sigma, clip, max_range)
        out[: w.shape[0]] = torch.from_numpy(w)
        d_count[0] = w.shape[0]

    def voxel_first_f64(self, points, voxel_size, max_range, out, d_out, scratch):
        assert points.dtype == out.dtype == torch.float64
        self.launches += 4
        w, status = restate_voxel_first(points.numpy(), voxel_size, max_range)
        out[: w.shape[0]] = torch.from_numpy(w)
        d_out[0], d_out[1] = w.shape[0], status

    def pc_tree(self, pts):
        self.launches += 12
        return pts.numpy().copy()

    def pc_nn(self, q, tree, dist, idx=None):
        """exact nearest neighbour by fp64 brute force in lb2_pc_nn's order, lowest index on ties, (+inf, -1) without a finite d²"""
        self.launches += 6
        d, j = metrics_reference.nn(q.numpy(), tree)
        dist[:] = torch.from_numpy(d)
        if idx is not None:
            idx[:] = torch.from_numpy(j.astype(np.int32))


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake (host-logic tests only); returns the handle"""
    h = FakeRefineHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
