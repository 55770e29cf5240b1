"""Records what the reference's evaluation metrics report on a seeded, scan-like pair of clouds, so lidiff_b200.metrics can be
compared against them without the reference's source tree:

    python tests/golden/make_metrics_goldens.py REF        # REF = a checkout of the reference -> tests/golden/metrics_reference.json

The reference's `lidiff/utils/metrics.py` and `lidiff/utils/histogram_metrics.py` run unchanged on the open3d shim on the CPU
(numpy's histogramdd; the 0.1 m IoU grid takes about 16 GB of host memory once).  Three stand-ins: `metrics.py` uses `torch.Tensor`
without importing torch, so torch is injected; `histogram_metrics.py` imports matplotlib.pyplot for a visualisation branch the
metrics never take, so a stub module is installed; and open3d's compute_point_cloud_distance is an exact fp64 k-d tree search,
which the shim's CPU branch (a bucketed search in fp32) does not always reproduce (on this pair it returns a farther neighbour for
367 of the 119 000 predicted points, by up to 4.7 mm), so the shim's method is replaced by scipy's exact cKDTree for the
recording.  The clouds are regenerated from the seed by `metrics_pair()`; only the results are stored.
"""
import importlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

PR_ARGS = (0.05, 0.1, 100)             # PrecisionRecall(0.05, 2 * 0.05, 100) as eval_path.py builds it
VOXEL_SIZES = [0.5, 0.2, 0.1]


def metrics_pair(seed=11):
    """(gt ~200k, pred ~120k) float64 clouds shaped like a completed scan and its ground truth: two synthetic scans for the gt,
    a noisy subset plus spurious points for the prediction, both with points beyond +-50 m and points exactly on the
    histogram bin edges (values of np.linspace(-50, 50, bins + 1) at every voxel size, and +-50 itself)"""
    from lidiff_b200.synth import synthetic_scan
    g = np.random.default_rng(seed)
    gt = np.concatenate([synthetic_scan(seed, beams=64, azimuths=2048), synthetic_scan(seed + 1, beams=32, azimuths=2048)])
    keep = g.choice(gt.shape[0], 120_000 - 6_000, replace=False)
    pred = gt[np.sort(keep)] + g.normal(0.0, 0.04, (keep.shape[0], 3))
    pred = np.concatenate([pred, g.uniform(-40, 40, (2_000, 3)) * [1, 1, 0.1]])

    def far(n):                         # beyond the +-50 m histogram range on at least one axis
        r, a = g.uniform(55, 150, n), g.uniform(-np.pi, np.pi, n)
        return np.stack([r * np.cos(a), r * np.sin(a), g.uniform(-3, 3, n)], 1)

    def on_edges(n):
        cols = []
        for _ in range(3):
            vs = VOXEL_SIZES[g.integers(0, 3)]
            edges = np.linspace(-50.0, 50.0, int(2 * 50.0 / vs) + 1)
            cols.append(edges[g.integers(0, edges.shape[0], n)])
        p = np.stack(cols, 1)
        p[: n // 8, g.integers(0, 3)] = g.choice([-50.0, 50.0], n // 8)
        return p

    gt = np.concatenate([gt, far(1_500), on_edges(2_000)])
    pred = np.concatenate([pred, far(1_000), on_edges(1_000), gt[-1_000:]])        # some edge points shared with the gt
    return np.ascontiguousarray(gt), np.ascontiguousarray(pred)


def main(ref):
    import torch
    import lidiff_b200.shims as sh
    sh.install()
    import open3d as o3d
    from scipy.spatial import cKDTree

    def exact_distance(self, target):
        return cKDTree(np.asarray(target.points, dtype=np.float64)).query(np.asarray(self.points, dtype=np.float64))[0]
    o3d.geometry.PointCloud.compute_point_cloud_distance = exact_distance
    sys.modules.setdefault("matplotlib", types.ModuleType("matplotlib"))
    sys.modules.setdefault("matplotlib.pyplot", types.ModuleType("matplotlib.pyplot"))
    sys.path.insert(0, ref)
    for k in [k for k in sys.modules if k == "lidiff" or k.startswith("lidiff.")]:
        sys.modules.pop(k)
    metrics = importlib.import_module("lidiff.utils.metrics")
    metrics.torch = torch
    hist = importlib.import_module("lidiff.utils.histogram_metrics")
    gt, pred = metrics_pair()
    pg, pp = o3d.geometry.PointCloud(gt), o3d.geometry.PointCloud(pred)
    rm, cd = metrics.RMSE(), metrics.ChamferDistance()
    rm.update(pg, pp)
    cd.update(pg, pp)
    pr = metrics.PrecisionRecall(*PR_ARGS)
    pr.update(pg, pp)
    p_all, r_all, f_all = pr.compute_at_all_thresholds()
    iou = metrics.CompletionIoU(VOXEL_SIZES)
    iou.update(pg, pp)
    out = {
        "seed": 11, "n_gt": int(gt.shape[0]), "n_pred": int(pred.shape[0]),
        "rmse": [float(v) for v in rm.compute()], "chamfer": [float(v) for v in cd.compute()],
        "pr_args": list(PR_ARGS), "precision": [float(v) for v in p_all], "recall": [float(v) for v in r_all],
        "f1": [float(v) for v in f_all], "auc": [float(v) for v in pr.compute_auc()],
        "iou_conf": {str(v): [int(c) for c in iou.conf_matrix[i]] for i, v in enumerate(VOXEL_SIZES)},
        "iou": {str(k): float(v) for k, v in iou.compute().items()},
        "jsd_3d": float(hist.compute_hist_metrics(pg, pp, bev=False)),
        "jsd_bev": float(hist.compute_hist_metrics(pg, pp, bev=True)),
    }
    json.dump(out, open(os.path.join(HERE, "metrics_reference.json"), "w"), indent=1)
    print({k: v for k, v in out.items() if k not in ("precision", "recall", "f1")})


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
