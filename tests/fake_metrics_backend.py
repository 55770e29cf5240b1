"""TEST INFRASTRUCTURE: CPU stand-ins (scipy / numpy) for the evaluation-metric methods of `lidiff_b200._lib.Handle`, on top of
the CPU fake of tests/fake_backend.py, so the host logic of lidiff_b200.metrics and the eval_path CLI can be exercised without a GPU.
Tests install it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_backend
import metrics_reference


class _Tree:
    """the reference cloud (`data`, every row) and a cKDTree over its finite rows (`kd`, None without any; `live` their indices)"""

    def __init__(self, pts):
        from scipy.spatial import cKDTree
        self.data = pts
        self.live = np.nonzero(np.isfinite(pts).all(1))[0]
        self.kd = cKDTree(pts[self.live]) if self.live.shape[0] else None


class FakeMetricsHandle(fake_backend.FakeHandle):
    def pc_tree(self, pts):
        self.launches += 12
        return _Tree(pts.numpy())

    def pc_nn(self, q, tree, dist, idx=None):
        """lb2_pc_nn's contract: a query without a finite squared distance (non-finite, no finite reference point, overflow)
        gets (+inf, -1)"""
        self.launches += 6
        qn = q.numpy()
        d, j = np.full(qn.shape[0], np.inf), np.full(qn.shape[0], -1, np.int64)
        ok = np.isfinite(qn).all(1)
        if tree.kd is not None and ok.any():
            kd, kj = tree.kd.query(qn[ok], k=1)
            found = kd < np.inf                                      # cKDTree: inf and index n for no neighbour
            d[np.nonzero(ok)[0][found]] = kd[found]
            j[np.nonzero(ok)[0][found]] = tree.live[kj[found]]
        dist[:] = torch.from_numpy(d)
        if idx is not None:
            idx[:] = torch.from_numpy(j.astype(np.int32))

    @staticmethod
    def _bins(pts, edges):
        """np.histogramdd's cell of every point (C order), -1 outside the range"""
        e = edges.numpy()
        nb = e.shape[0] - 1
        b = np.searchsorted(e, pts.numpy(), side="right") - 1
        b[pts.numpy() == e[-1]] = nb - 1
        ok = ((b >= 0) & (b < nb)).all(1)
        return np.where(ok, (b[:, 0] * nb + b[:, 1]) * nb + b[:, 2], -1), nb

    def voxel_occupancy(self, pts, edges, bits=None, counts=None, n_in=None):
        self.launches += 1
        cell, nb = self._bins(pts, edges)
        cell = cell[cell >= 0]
        if bits is not None:
            w = np.zeros(bits.shape[0], np.uint32)
            np.bitwise_or.at(w, cell >> 5, (np.uint32(1) << (cell & 31).astype(np.uint32)))
            bits[:] = torch.from_numpy(w.view(np.int32))
        if counts is not None:
            counts[:] = torch.from_numpy(np.bincount(cell, minlength=nb ** 3).astype(np.int32))
        if n_in is not None:
            n_in[0] = int(cell.shape[0])

    @staticmethod
    def _unpack(bits, nbits):
        return np.unpackbits(bits.numpy().view(np.uint8), bitorder="little")[:nbits].astype(bool)

    def occupancy_confusion(self, bits_gt, bits_pred, nbits, out):
        self.launches += 1
        a, b = self._unpack(bits_gt, nbits), self._unpack(bits_pred, nbits)
        out[:] = torch.tensor([(a & b).sum(), (a & ~b).sum(), (~a & b).sum()])

    def occupancy_bev(self, bits, bins, bev):
        self.launches += 1
        bev[:] = torch.from_numpy(self._unpack(bits, bins ** 3).reshape(bins * bins, bins).sum(1).astype(np.int32))

    def jsd(self, hist_a, hist_b, out):
        from scipy.spatial.distance import jensenshannon
        self.launches += 3
        a, b = hist_a.numpy().view(np.uint32).astype(np.float64), hist_b.numpy().view(np.uint32).astype(np.float64)
        out[0] = float(jensenshannon(a / a.sum(), b / b.sum())) if a.sum() and b.sum() else float("nan")

    def dist_stats(self, dist, thresholds, sum_out, counts_out):
        """the kernel's order and its binary search, which counts correctly only for ascending, NaN-free thresholds"""
        self.launches += 2
        d = dist.numpy()
        sum_out[0] = metrics_reference.ordered_sum(d)
        counts_out[:] = torch.from_numpy(metrics_reference.ds_kernel_counts(d, thresholds.numpy()))


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake with the metric stand-ins (host-logic tests only)"""
    from lidiff_b200 import _lib
    h = FakeMetricsHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
