"""Evaluation metrics of completed scans on the GPU — the counterpart of the reference's `lidiff/utils/metrics.py` (RMSE,
ChamferDistance, PrecisionRecall, CompletionIoU) and `lidiff/utils/histogram_metrics.py` (compute_hist_metrics), with the same
classes, methods and semantics, computed by the lidiff_b200 CUDA library:

  * nearest-neighbour distances: exact fp64 1-NN over a Morton-sorted box hierarchy (lb2_pc_tree_build / lb2_pc_nn), the
    counterpart of open3d's compute_point_cloud_distance;
  * occupancy and counts: np.histogramdd's binning over [-50, 50]^3, bit for bit (lb2_voxel_occupancy), as bitsets, so the 0.1 m
    grid takes 125 MB instead of numpy's dense 8 GB;
  * reductions: IoU confusion counts, BEV histograms, Jensen-Shannon distance, distance sums and threshold counts, all
    deterministic (integer counts, fixed-order fp64 sums).

`evaluate_scan(gt, pred)` computes each direction's distances once and the occupancy once per voxel size and returns a
`ScanRecord`; the accumulators consume records with `add`, and their `update(gt, pred)` evaluates what they need.  Points may be
numpy arrays, torch tensors on any device, or open3d-shim PointClouds.  There is no CPU fallback.
"""
from __future__ import annotations

import dataclasses

import numpy as np
import scipy.integrate
import torch

from . import _lib
from .rowsum import GatherRows

MAX_RANGE = 50.0                        # histogram range [-MAX_RANGE, MAX_RANGE] on every axis (metrics.py:88)
JSD_VOXEL = 0.5                         # histogram_metrics.py:48-49
VOXEL_SIZES = (0.5, 0.2, 0.1)           # CompletionIoU default
PR_ARGS = (0.05, 0.1, 100)              # PrecisionRecall(0.05, 2 * 0.05, 100) of eval_path.py


def _xyz(x) -> torch.Tensor | np.ndarray:
    if hasattr(x, "points") and not isinstance(x, (np.ndarray, torch.Tensor)):
        x = np.asarray(x.points)
    if isinstance(x, torch.Tensor):
        x = x.detach()
    if x.ndim != 2 or x.shape[1] < 3:
        raise ValueError(f"expected an (n, 3) point array, got shape {tuple(x.shape)}")
    return x[:, :3]


def _points(x, device) -> torch.Tensor:
    """(n, 3) contiguous fp64 tensor on `device`"""
    return torch.as_tensor(_xyz(x)).to(device=device, dtype=torch.float64).contiguous()


def voxel_bins(voxel_size: float) -> int:
    return int(2 * MAX_RANGE / voxel_size)


def voxel_edges(voxel_size: float) -> np.ndarray:
    """np.histogramdd's bin edges for range [-50, 50] (np.linspace, bins + 1 values)"""
    return np.linspace(-MAX_RANGE, MAX_RANGE, voxel_bins(voxel_size) + 1)


def nn_distance(query, ref, return_index: bool = False, device="cuda"):
    """distance of every query point to its nearest point of `ref` (fp64 torch tensor on the device; open3d's
    compute_point_cloud_distance), and with return_index the index of that point (lowest index on equal distances)"""
    h = _lib.get_handle(device)
    q, r = _points(query, h.device), _points(ref, h.device)
    if r.shape[0] == 0:
        raise ValueError("nn_distance: empty reference cloud")
    dist = torch.empty(q.shape[0], dtype=torch.float64, device=h.device)
    idx = torch.empty(q.shape[0], dtype=torch.int32, device=h.device) if return_index else None
    if q.shape[0]:
        h.pc_nn(q, h.pc_tree(r), dist, idx)
    return (dist, idx) if return_index else dist


@dataclasses.dataclass
class ScanRecord:
    """what one scan contributes to the metrics (all host values)"""
    n_gt: int
    n_pred: int
    sum_pred_to_gt: float = float("nan")            # sums of the nearest-neighbour distances per direction
    sum_gt_to_pred: float = float("nan")
    thresholds: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0))
    cnt_pred_to_gt: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0, np.int64))   # number of distances < t
    cnt_gt_to_pred: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0, np.int64))
    voxel_sizes: tuple = ()
    conf: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros((0, 3), np.uint64))      # (tp, fn, fp) per voxel size
    jsd_3d: float = float("nan")
    jsd_bev: float = float("nan")

    @property
    def mean_pred_to_gt(self) -> float:
        return self.sum_pred_to_gt / self.n_pred

    @property
    def mean_gt_to_pred(self) -> float:
        return self.sum_gt_to_pred / self.n_gt


def evaluate_scan(gt, pred, thresholds=None, voxel_sizes=VOXEL_SIZES, distances: str = "both", hist: bool = True, device="cuda",
                  events: dict | None = None) -> ScanRecord:
    """Every metric of one (ground truth, prediction) pair in one pass: nearest-neighbour distances per direction (`distances`:
    "both", "pred" = prediction -> gt only, or "none"), their sums and counts below `thresholds` (default: np.linspace(*PR_ARGS)),
    IoU confusion counts at `voxel_sizes`, and with `hist` the 3D and BEV Jensen-Shannon distances at 0.5 m.  One host
    synchronisation at the end.  `events`, if given, receives CUDA event pairs per phase (benchmarking).
    Raises ValueError for an empty cloud, or when a histogram is needed and a cloud has no point inside [-50, 50]^3."""
    h = _lib.get_handle(device)
    dev = h.device
    g, p = _points(gt, dev), _points(pred, dev)
    if g.shape[0] == 0 or p.shape[0] == 0:
        raise ValueError(f"evaluate_scan: empty cloud (gt {g.shape[0]} points, prediction {p.shape[0]} points)")
    thr_np = np.linspace(*PR_ARGS) if thresholds is None else np.asarray(thresholds, dtype=np.float64)
    rec = ScanRecord(n_gt=int(g.shape[0]), n_pred=int(p.shape[0]), thresholds=thr_np, voxel_sizes=tuple(voxel_sizes))

    def mark(name):
        if events is not None and dev.type == "cuda":
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            events.setdefault(name, []).append(ev)

    dirs = {"both": (("pred_to_gt", p, g), ("gt_to_pred", g, p)), "pred": (("pred_to_gt", p, g),), "none": ()}[distances]
    thr = torch.as_tensor(thr_np, device=dev)
    sums = torch.zeros(len(dirs), dtype=torch.float64, device=dev)
    cnts = torch.zeros((len(dirs), thr_np.shape[0]), dtype=torch.int64, device=dev)
    for k, (_, q, r) in enumerate(dirs):
        mark("nn_build")
        tree = h.pc_tree(r)
        mark("nn_query")
        dist = torch.empty(q.shape[0], dtype=torch.float64, device=dev)
        h.pc_nn(q, tree, dist)
        h.dist_stats(dist, thr, sums[k:k + 1], cnts[k])
        mark("nn_end")

    sizes = list(voxel_sizes) + ([JSD_VOXEL] if hist and JSD_VOXEL not in voxel_sizes else [])
    conf = torch.zeros((len(sizes), 3), dtype=torch.int64, device=dev)
    n_in = torch.zeros((len(sizes), 2), dtype=torch.int64, device=dev)
    jsd = torch.full((2,), float("nan"), dtype=torch.float64, device=dev)
    for k, vs in enumerate(sizes):
        mark(f"occupancy_{vs}")
        bins = voxel_bins(vs)
        edges = torch.as_tensor(voxel_edges(vs), device=dev)
        words = (bins ** 3 + 31) // 32
        want_hist = hist and vs == JSD_VOXEL
        bits = [torch.empty(words, dtype=torch.int32, device=dev) for _ in range(2)]
        counts = [torch.empty(bins ** 3, dtype=torch.int32, device=dev) if want_hist else None for _ in range(2)]
        for c, cloud in enumerate((g, p)):
            h.voxel_occupancy(cloud, edges, bits[c], counts[c], n_in[k, c:c + 1])
        h.occupancy_confusion(bits[0], bits[1], bins ** 3, conf[k])
        if want_hist:
            mark("jsd")
            h.jsd(counts[0], counts[1], jsd[0:1])
            bev = [torch.empty(bins * bins, dtype=torch.int32, device=dev) for _ in range(2)]
            for c in range(2):
                h.occupancy_bev(bits[c], bins, bev[c])
            h.jsd(bev[0], bev[1], jsd[1:2])
        mark("occupancy_end")

    sums, cnts, conf, n_in, jsd = (t.cpu().numpy() for t in (sums, cnts, conf, n_in, jsd))       # the one synchronisation
    if len(sizes) and (n_in == 0).any():
        raise ValueError("evaluate_scan: a cloud has no point inside the [-50, 50] m histogram range")
    for k, (name, _, _) in enumerate(dirs):
        setattr(rec, f"sum_{name}", float(sums[k]))
        setattr(rec, f"cnt_{name}", cnts[k].astype(np.int64))
    rec.conf = conf[: len(voxel_sizes)].astype(np.uint64)
    if hist:
        rec.jsd_3d, rec.jsd_bev = float(jsd[0]), float(jsd[1])
    return rec


def compute_hist_metrics(pcd_gt, pcd_pred, bev: bool = False, device="cuda") -> float:
    """histogram_metrics.compute_hist_metrics: Jensen-Shannon distance of the 0.5 m histograms (bev: occupancy summed over z)"""
    rec = evaluate_scan(pcd_gt, pcd_pred, thresholds=(), voxel_sizes=(), distances="none", hist=True, device=device)
    return rec.jsd_bev if bev else rec.jsd_3d


class RMSE:
    """mean prediction -> gt distance per scan; compute() = (mean, std) over scans"""

    def __init__(self):
        self.dists = []

    def update(self, gt_pcd, pt_pcd):
        self.add(evaluate_scan(gt_pcd, pt_pcd, thresholds=(), voxel_sizes=(), distances="pred", hist=False))

    def add(self, rec: ScanRecord):
        self.dists.append(rec.mean_pred_to_gt)

    def reset(self):
        self.dists = []

    def compute(self):
        d = np.array(self.dists)
        return d.mean(), d.std()


class ChamferDistance:
    """per scan (mean gt -> prediction + mean prediction -> gt) / 2; compute() = (mean, std) over scans"""

    def __init__(self):
        self.dists = []

    def update(self, gt_pcd, pt_pcd):
        self.add(evaluate_scan(gt_pcd, pt_pcd, thresholds=(), voxel_sizes=(), hist=False))

    def add(self, rec: ScanRecord):
        self.dists.append((rec.mean_gt_to_pred + rec.mean_pred_to_gt) / 2)

    def reset(self):
        self.dists = []

    def compute(self):
        d = np.array(self.dists)
        return d.mean(), d.std()


class PrecisionRecall:
    """precision (share of predicted points closer than t to the gt) and recall (share of gt points closer than t to the
    prediction) in percent at np.linspace(min_t, max_t, num) thresholds, F-score 0 when either is 0; averaged over scans"""

    def __init__(self, min_t, max_t, num):
        self.thresholds = np.linspace(min_t, max_t, num)
        self.reset()

    def update(self, gt_pcd, pt_pcd):
        self.add(evaluate_scan(gt_pcd, pt_pcd, thresholds=self.thresholds, voxel_sizes=(), hist=False))

    def add(self, rec: ScanRecord):
        if not np.array_equal(rec.thresholds, self.thresholds):
            raise ValueError("PrecisionRecall.add: the record was evaluated at other thresholds")
        p = 100 / rec.n_pred * rec.cnt_pred_to_gt
        r = 100 / rec.n_gt * rec.cnt_gt_to_pred
        with np.errstate(invalid="ignore", divide="ignore"):
            f = np.where((p == 0) | (r == 0), 0.0, 2 * p * r / (p + r))
        self.pr.append(p)
        self.re.append(r)
        self.f1.append(f)

    def reset(self):
        self.pr, self.re, self.f1 = [], [], []

    def compute_at_all_thresholds(self):
        """per-threshold means over the scans (sequential sums, as lists)"""
        return tuple([sum(float(s[k]) for s in rows) / len(rows) for k in range(len(self.thresholds))] for rows in (self.pr, self.re, self.f1))

    def find_nearest_threshold(self, value):
        return self.thresholds[np.abs(self.thresholds - value).argmin()]

    def compute_at_threshold(self, threshold):
        k = int(np.abs(self.thresholds - threshold).argmin())
        pr, re, f1 = self.compute_at_all_thresholds()
        return pr[k], re[k], f1[k], self.thresholds[k]

    def compute_auc(self):
        """areas under the precision / recall / F curves (Simpson's rule) over the area of a perfect predictor"""
        dx = self.thresholds[1] - self.thresholds[0]
        perfect = scipy.integrate.simpson(np.ones_like(self.thresholds), dx=dx)
        return tuple(scipy.integrate.simpson(v, dx=dx) / perfect for v in self.compute_at_all_thresholds())


class CompletionIoU:
    """occupancy IoU of the [-50, 50]^3 voxel grids at each voxel size, tp / (tp + fn + fp) over counts accumulated across scans"""

    def __init__(self, voxel_sizes=list(VOXEL_SIZES)):
        self.voxel_sizes = list(voxel_sizes)
        self.reset()

    def update(self, gt, pred):
        self.add(evaluate_scan(gt, pred, thresholds=(), voxel_sizes=self.voxel_sizes, distances="none", hist=False))

    def add(self, rec: ScanRecord):
        for i, vs in enumerate(self.voxel_sizes):
            self.conf_matrix[i] += rec.conf[list(rec.voxel_sizes).index(vs)].astype(np.uint64)

    def reset(self):
        self.conf_matrix = np.zeros((len(self.voxel_sizes), 3), dtype=np.uint64)

    def compute(self):
        return {vs: self.conf_matrix[i][0] / (self.conf_matrix[i][0] + self.conf_matrix[i][1] + self.conf_matrix[i][2] + 1e-15)
                for i, vs in enumerate(self.voxel_sizes)}


# ---- per-scan records across ranks: a record travels as float32 rows (the raw bytes of its fp64 / int64 fields), so that
# sharding.gather_scans carries it unchanged and rank 0 decodes exactly what the other ranks computed --------------------------------
def record_to_rows(rec: ScanRecord) -> torch.Tensor:
    nt, nv = rec.thresholds.shape[0], len(rec.voxel_sizes)
    vals = np.concatenate([np.array([rec.n_gt, rec.n_pred, nt, nv], np.float64),
                           np.array([rec.sum_pred_to_gt, rec.sum_gt_to_pred, rec.jsd_3d, rec.jsd_bev]),
                           rec.thresholds, np.asarray(rec.voxel_sizes, np.float64),
                           rec.cnt_pred_to_gt.astype(np.int64).view(np.float64), rec.cnt_gt_to_pred.astype(np.int64).view(np.float64),
                           rec.conf.astype(np.uint64).reshape(-1).view(np.float64)])
    words = vals.view(np.float32)
    words = np.concatenate([words, np.zeros((-words.shape[0]) % 3, np.float32)])
    return torch.from_numpy(words.reshape(-1, 3).copy())


def record_from_rows(rows: torch.Tensor) -> ScanRecord:
    words = rows.detach().cpu().contiguous().numpy().astype(np.float32, copy=False).reshape(-1)
    v = words[: words.shape[0] - words.shape[0] % 2].view(np.float64)
    n_gt, n_pred, nt, nv = (int(x) for x in v[:4])
    o = 8
    take = lambda k: v[o:o + k]
    thr = take(nt).copy(); o += nt
    vs = tuple(float(x) for x in take(nv)); o += nv
    c_pg = take(nt).view(np.int64).copy(); o += nt
    c_gp = take(nt).view(np.int64).copy(); o += nt
    conf = take(3 * nv).view(np.uint64).reshape(nv, 3).copy()
    return ScanRecord(n_gt, n_pred, float(v[4]), float(v[5]), thr, c_pg, c_gp, vs, conf, float(v[6]), float(v[7]))


def _nn_sq_dist(q: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """((q - r[idx])**2).sum(-1) in q's dtype, idx = the exact (fp64) nearest point of r to every row of q, lowest index on ties.
    Differentiable in q and r; the gradient of r[idx] is summed per row of r in query order (rowsum.GatherRows), without atomics."""
    with torch.no_grad():
        _, idx = nn_distance(q, r, return_index=True, device=q.device)
    return ((q - GatherRows.apply(r, idx.long())) ** 2).sum(-1)


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None, batch_reduction="mean",
                     point_reduction="mean", norm=2):
    """pytorch3d.loss.chamfer_distance (pytorch3d 0.7.1) with its defaults, on (B, P, 3) tensors on the GPU: (loss, None).

    Every point's nearest neighbour in the other cloud is exact (lb2_pc_nn on fp64 coordinates, lowest index on ties), and its
    squared distance is recomputed in the clouds' dtype as ((q - p[idx])**2).sum(-1); pytorch3d's fp32 brute force can pick the
    other point of a near-tie, a few fp32 ulps apart (DESIGN.md §5).  The reductions are pytorch3d's torch ops in its order: the
    per-cloud .sum(1), / lengths, .sum() / B, cham_x + cham_y.  Any other argument raises NotImplementedError.

    The loss is differentiable in x and y: the neighbour indices are fixed by the forward (as pytorch3d's backward uses its knn
    indices), and the gradient that the cham_y term sends to x[idx_y] is summed per point of x in a fixed order."""
    if any(a is not None for a in (x_lengths, y_lengths, x_normals, y_normals, weights)) or batch_reduction != "mean" or \
            point_reduction != "mean" or norm != 2:
        raise NotImplementedError("chamfer_distance: only pytorch3d's defaults (no lengths / normals / weights, mean reductions, "
                                  "norm 2) are implemented")
    if not (isinstance(x, torch.Tensor) and isinstance(y, torch.Tensor)) or x.dim() != 3 or y.dim() != 3 or x.shape[2] != 3 or \
            y.shape[2] != 3:
        raise ValueError(f"chamfer_distance: expected (B, P, 3) tensors, got {tuple(getattr(x, 'shape', ()))} and "
                         f"{tuple(getattr(y, 'shape', ()))}")
    if x.shape[0] != y.shape[0]:
        raise ValueError("chamfer_distance: x and y must have the same batch dimension")
    if x.shape[1] == 0 or y.shape[1] == 0:
        raise ValueError("chamfer_distance: empty point cloud")
    y = y.to(x.device)
    n = x.shape[0]
    cham_x = torch.stack([_nn_sq_dist(x[b], y[b]) for b in range(n)])          # (B, P1)
    cham_y = torch.stack([_nn_sq_dist(y[b], x[b]) for b in range(n)])          # (B, P2)
    x_lengths = torch.full((n,), x.shape[1], dtype=torch.int64, device=x.device)
    y_lengths = torch.full((n,), y.shape[1], dtype=torch.int64, device=x.device)
    cham_x = cham_x.sum(1)
    cham_y = cham_y.sum(1)
    cham_x /= x_lengths.clamp(min=1)
    cham_y /= y_lengths.clamp(min=1)
    cham_x = cham_x.sum()
    cham_y = cham_y.sum()
    div = max(n, 1)
    cham_x /= div
    cham_y /= div
    return cham_x + cham_y, None
