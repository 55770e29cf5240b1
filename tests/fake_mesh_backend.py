"""TEST INFRASTRUCTURE: CPU stand-ins for the mesh-sampling methods of `lidiff_b200._lib.Handle` (mesh_sample_prepare,
mesh_sample_points) from the numpy restatement of tests/mesh_reference.py, with the MT19937 word stand-in of
tests/fake_rng_backend.py and the metric stand-ins of tests/fake_metrics_backend.py, so the host logic of lidiff_b200.mesh, the
open3d shim's TriangleMesh and `eval_path --mesh` runs without a GPU.  Tests install it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_metrics_backend
import mesh_reference as MR
from fake_rng_backend import FakeRngMixin
from lidiff_b200 import _lib

_INFO = np.dtype([("surface_area", "<f8"), ("last_count", "<i8"), ("status", "<i4"), ("pad", "<i4")])


class FakeMeshHandle(FakeRngMixin, fake_metrics_backend.FakeMetricsHandle):
    def mesh_sample_scratch(self, n_tris):
        return torch.zeros(max(24 * int(n_tris), 1), dtype=torch.uint8)

    def mesh_sample_prepare(self, verts, tris, n_points, area, info, scratch):
        """lb2_mesh_sample_prepare's contract: the status bits, the areas, S and the n_t (int64 at the start of scratch)"""
        assert verts.dtype == torch.float64 and tris.dtype == torch.int32 and area.shape[0] == tris.shape[0]
        self.launches += 5
        v, t = verts.numpy(), tris.numpy().astype(np.int64)
        rec = np.zeros(1, _INFO)
        bad = ((t < 0) | (t >= v.shape[0])).any(1)
        if bad.any():
            rec["status"] |= _lib.MESH_BAD_INDEX
        ok = np.flatnonzero(~bad)
        if not np.isfinite(v[t[ok]]).all():
            rec["status"] |= _lib.MESH_NON_FINITE
        a = np.zeros(t.shape[0])
        a[ok] = MR.areas(v, t[ok])
        area[:] = torch.from_numpy(a)
        s = MR.surface_area(a)
        rec["surface_area"] = s
        if not (0.0 < s < np.inf):
            rec["status"] |= _lib.MESH_BAD_AREA
        else:
            with np.errstate(invalid="ignore"):
                n_t = MR.counts(a, n_points)
            scratch[:8 * n_t.shape[0]] = torch.from_numpy(n_t.view(np.uint8))
            rec["last_count"] = n_t[-1]
            if n_t[-1] != n_points:
                rec["status"] |= _lib.MESH_BAD_COUNT
        info[:] = torch.from_numpy(rec.view(np.uint8).copy())

    def mesh_sample_points(self, verts, tris, scratch, words, n_points, out):
        self.launches += 1
        w = words[:4 * n_points].numpy().view(np.uint32)
        out[:] = torch.from_numpy(MR.sample(verts.numpy(), tris.numpy(), n_points, w))


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake with the mesh stand-ins (host-logic tests only)"""
    h = FakeMeshHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
