"""TEST INFRASTRUCTURE: CPU stand-ins for the scene-completion grid methods of `lidiff_b200._lib.Handle` (ssc_grid_count,
ssc_grid_points, ssc_voxelize, ssc_confusion) from the numpy restatement of tests/ssc_reference.py, on top of the metric stand-ins
of tests/fake_metrics_backend.py, so the host logic of lidiff_b200.ssc and `eval_path --voxels / --ssc` runs without a GPU.
Tests install it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_metrics_backend
import ssc_reference as SR
from lidiff_b200 import _lib


class FakeSSCHandle(fake_metrics_backend.FakeMetricsHandle):
    def __init__(self):
        super().__init__()
        self._occ = {}

    def ssc_scratch(self, n_grids):
        return torch.zeros(max(int(n_grids) * (8 * SR.N_WORDS + 8), 1), dtype=torch.uint8)

    def _occupancy(self, grids, kind):
        g = grids.numpy()
        if kind == _lib.SSC_LABELS:
            return [SR.occupied(r.view(np.uint16)) for r in g]
        return [SR.unpack(r.view(np.uint32)) for r in g]

    def ssc_grid_count(self, grids, kind, n_grids, offsets, scratch):
        assert grids.shape[0] == n_grids and grids.is_contiguous()
        self.launches += 3
        occ = self._occupancy(grids, kind)
        self._occ[scratch.data_ptr()] = occ
        offsets[:] = torch.from_numpy(np.concatenate([[0], np.cumsum([o.sum() for o in occ])]).astype(np.int64))

    def ssc_grid_points(self, n_grids, offsets, scratch, out):
        self.launches += 1
        occ = self._occ.pop(scratch.data_ptr())
        assert len(occ) == n_grids
        out[:] = torch.from_numpy(np.concatenate([SR.centres(o) for o in occ]))

    def ssc_voxelize(self, pts, offsets, n_grids, bits, info):
        self.launches += 1
        p, off = pts.numpy(), offsets.numpy()
        rec = np.zeros((n_grids, 2), np.int64)
        for g in range(n_grids):
            w, rec[g, 0], rec[g, 1] = SR.voxelize(p[off[g]:off[g + 1]])
            bits[g] = torch.from_numpy(w.view(np.int32))
        info[:] = torch.from_numpy(rec.view(np.uint8).reshape(-1).copy())

    def ssc_confusion(self, pred_bits, gt_labels, invalid, n_grids, out):
        self.launches += 1
        for g in range(n_grids):
            inv = None if invalid is None else invalid[g].numpy().view(np.uint32)
            out[g] = torch.tensor(SR.confusion(pred_bits[g].numpy().view(np.uint32), gt_labels[g].numpy().view(np.uint16), inv))


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake with the SSC stand-ins (host-logic tests only)"""
    h = FakeSSCHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
