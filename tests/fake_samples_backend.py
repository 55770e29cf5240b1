"""TEST INFRASTRUCTURE: a numpy stand-in for the sample methods of `lidiff_b200._lib.Handle` (lb2_select_points /
lb2_viewpoint_filter), on top of the CPU fake of tests/fake_backend.py, so the host logic of lidiff_b200.datasets can be exercised
without a GPU.  `restate_select` / `restate_viewpoint` restate the kernels' documented arithmetic in numpy (every operation rounded,
no FMA) and are also the yardstick of the GPU tests.  Tests install it by monkeypatching `_lib.get_handle`, and the dataset's
farthest point sampling with the oracle's numpy one."""
import numpy as np
import torch

import fake_backend
from lidiff_b200 import _lib

AXIS_LIMIT = 1 << 21


def restate_select(points, labels, desc):
    """the fp64 (m, 3) rows lb2_select_points keeps, in input order"""
    p = np.asarray(points)
    x, y, z = (p[:, j].astype(np.float64) for j in range(3))
    keep = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
    if labels is not None:
        lab = np.asarray(labels).view(np.uint32) & np.uint32(0xFFFF)
        keep &= (lab > 1) & (lab < 252)
    c = [float(v) for v in desc.center]
    with np.errstate(invalid="ignore", over="ignore"):
        if desc.range_mode == _lib.RANGE_FP32:
            f = np.float32
            dx, dy, dz = x.astype(f) - f(c[0]), y.astype(f) - f(c[1]), z.astype(f) - f(c[2])
            d = np.sqrt((dx * dx + dy * dy) + dz * dz)
            keep &= (d > f(desc.r_min)) & (d < f(desc.r_max))
        elif desc.range_mode == _lib.RANGE_FP64:
            dx, dy, dz = x - c[0], y - c[1], z - c[2]
            d = np.sqrt((dx * dx + dy * dy) + dz * dz)
            keep &= (d > desc.r_min) & (d < desc.r_max)
        if desc.has_transform:
            m = np.array(list(desc.transform)).reshape(3, 4)
            x, y, z = (((m[k, 0] * x + m[k, 1] * y) + m[k, 2] * z) + m[k, 3] for k in range(3))
        if desc.has_z_min:
            keep &= z > desc.z_min
    return np.stack([x, y, z], 1)[keep]


def restate_viewpoint(part, full, voxel):
    """(kept mask of `full`, status) of lb2_viewpoint_filter: the open3d shim's VoxelGrid with cell indices keyed in [0, 2^21)"""
    part, full = np.asarray(part, dtype=np.float64), np.asarray(full, dtype=np.float64)
    if len(part) == 0 or len(full) == 0:
        return np.zeros(len(full), bool), 0
    origin = part.min(0) - 0.5 * voxel
    with np.errstate(invalid="ignore"):
        cp, cf = np.floor((part - origin) / voxel), np.floor((full - origin) / voxel)
    ok_p = ((cp >= 0) & (cp < AXIS_LIMIT)).all(1)
    ok_f = ((cf >= 0) & (cf < AXIS_LIMIT)).all(1)
    enc = lambda c: (c[:, 0].astype(np.int64) * AXIS_LIMIT + c[:, 1].astype(np.int64)) * AXIS_LIMIT + c[:, 2].astype(np.int64)
    keys = enc(cp[ok_p])
    kf = np.zeros(len(full), np.int64)
    kf[ok_f] = enc(cf[ok_f])
    return ok_f & np.isin(kf, keys), int(not ok_p.all())


class FakeSamplesHandle(fake_backend.FakeHandle):
    def select_points_scratch(self, n):
        return torch.empty(16, dtype=torch.uint8)

    def viewpoint_filter_scratch(self, n_part, n_full):
        return torch.empty(16, dtype=torch.uint8)

    def select_points(self, points, labels, desc, out, d_count, scratch):
        assert points.dim() == 2 and points.shape[1] in (3, 4) and points.dtype in (torch.float32, torch.float64)
        self.launches += 3
        w = restate_select(points.numpy(), None if labels is None else labels.numpy(), desc)
        out[: w.shape[0]] = torch.from_numpy(w)
        d_count[0] = w.shape[0]

    def viewpoint_filter(self, part, full, voxel_size, out, d_out, scratch):
        assert part.dtype == full.dtype == out.dtype == torch.float64
        self.launches += 5
        keep, status = restate_viewpoint(part.numpy(), full.numpy(), voxel_size)
        out[: int(keep.sum())] = full[torch.from_numpy(keep)]
        d_out[0], d_out[1] = int(keep.sum()), status


def fps_sorted(points, n):
    from oracle.pipeline import farthest_point_sample
    return torch.from_numpy(farthest_point_sample(points.numpy(), int(n)))


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake and its farthest point sampling to the oracle's (host-logic tests only);
    returns the handle and the list of batch sizes the batched sampling was called with"""
    from lidiff_b200 import datasets
    h = FakeSamplesHandle()
    batched = []
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    monkeypatch.setattr(datasets, "farthest_point_sample", fps_sorted)

    def fps_batched(scans, n):
        batched.append(len(scans))
        return torch.stack([fps_sorted(s, n) for s in scans])
    monkeypatch.setattr(datasets, "farthest_point_sample_batched", fps_batched)
    return h, batched
