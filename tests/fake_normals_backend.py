"""TEST INFRASTRUCTURE: CPU stand-ins for the point-normal methods of `lidiff_b200._lib.Handle` (pc_knn, pc_normals), computed by
the numpy restatement of open3d's estimate_normals (tests/normals_oracle.py), on top of the metric stand-ins of
tests/fake_metrics_backend.py (whose pc_tree is a scipy cKDTree), so the host logic of lidiff_b200.normals, the open3d shim and the
completion CLI can be exercised without a GPU.  Tests install it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_metrics_backend
import normals_oracle


class FakeNormalsHandle(fake_metrics_backend.FakeMetricsHandle):
    def pc_knn(self, tree, n, k, idx, d2=None):
        if not 1 <= k <= 32:
            raise RuntimeError("lb2_pc_knn failed (-3): pc_knn: k > 32 is not supported")
        assert tree.data.shape[0] == n and tuple(idx.shape) == (n, min(k, n)) and idx.dtype == torch.int32
        self.launches += 1
        j, d = normals_oracle.knn(tree.data, k)
        idx[:] = torch.from_numpy(j.astype(np.int32))
        if d2 is not None:
            assert d2.dtype == torch.float64 and d2.shape == idx.shape
            d2[:] = torch.from_numpy(d)

    def pc_normals(self, pts, idx, normals):
        assert pts.dtype == torch.float64 and idx.dtype == torch.int32 and normals.dtype == torch.float64
        assert tuple(normals.shape) == (pts.shape[0], 3) and idx.shape[0] == pts.shape[0]
        self.launches += 1
        nrm, _, _ = normals_oracle.normals_from_idx(pts.numpy(), idx.numpy().astype(np.int64))
        normals[:] = torch.from_numpy(nrm)


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake with the normal stand-ins (host-logic tests only)"""
    from lidiff_b200 import _lib
    h = FakeNormalsHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
