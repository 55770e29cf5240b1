"""The evaluation-metric kernels and lidiff_b200.metrics on the GPU: exact fp64 nearest neighbours against scipy's cKDTree,
np.histogramdd-exact occupancy and counts, Jensen-Shannon distances against scipy, the reference's own results on a seeded pair
(tests/golden/metrics_reference.json, recorded by tests/golden/make_metrics_goldens.py), determinism, the open3d shim and the
eval_path CLI."""
import json
import os
import sys

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree
from scipy.spatial.distance import jensenshannon

from lidiff_b200 import metrics as M

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.gpu


def _scan_like(n, seed):
    from lidiff_b200.synth import synthetic_scan
    parts, k = [], 0
    while sum(p.shape[0] for p in parts) < n:
        parts.append(synthetic_scan(seed + k))
        k += 1
    return np.concatenate(parts)[:n]


def _check_nn(q, r):
    d, idx = M.nn_distance(q, r, return_index=True)
    d, idx = d.cpu().numpy(), idx.cpu().numpy()
    kd, kj = cKDTree(r).query(q, k=2)
    assert np.abs(d - kd[:, 0]).max() <= 1e-12
    unique = kd[:, 1] > kd[:, 0]                                        # a one-point cloud gives inf as the second distance
    assert np.array_equal(idx[unique], kj[unique, 0])
    # every returned index is at the returned distance
    assert np.abs(np.sqrt(((q - r[idx]) ** 2).sum(1)) - d).max() <= 1e-12
    return d, idx


def test_nn_scan_like_1m_by_600k():
    gt = _scan_like(1_000_000, 0)
    g = np.random.default_rng(1)
    pred = gt[g.choice(gt.shape[0], 600_000, replace=False)] + g.normal(0, 0.05, (600_000, 3))
    _check_nn(pred, gt)
    _check_nn(gt, pred)


def test_nn_duplicates_and_lattice_ties_take_the_lowest_index():
    g = np.random.default_rng(2)
    base = g.uniform(-5, 5, (3000, 3))
    r = np.concatenate([base, base[::-1], base[:500]])                  # every point three or two times
    q = np.concatenate([base[:1000], g.uniform(-6, 6, (2000, 3))])
    d, idx = M.nn_distance(q, r, return_index=True)
    d, idx = d.cpu().numpy(), idx.cpu().numpy()
    kd, _ = cKDTree(r).query(q)
    assert np.abs(d - kd).max() <= 1e-12
    first = {tuple(p): i for i, p in reversed(list(enumerate(r)))}
    assert all(idx[i] == first[tuple(q[i])] for i in range(1000))
    # lattice with exact ties: queries at cell centres are equidistant to 8 lattice points
    ax = np.arange(12, dtype=np.float64)
    lat = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    perm = g.permutation(lat.shape[0])
    lat = lat[perm]
    cq = np.stack(np.meshgrid(ax[:-1] + 0.5, ax[:-1] + 0.5, ax[:-1] + 0.5, indexing="ij"), -1).reshape(-1, 3)
    d, idx = M.nn_distance(cq, lat, return_index=True)
    full = np.sqrt(((cq[:, None, :] - lat[None]) ** 2).sum(-1))
    want = np.argmin(np.where(full == full.min(1, keepdims=True), np.arange(lat.shape[0])[None], 1 << 30), 1)
    assert np.array_equal(idx.cpu().numpy(), want)
    assert np.abs(d.cpu().numpy() - full.min(1)).max() <= 1e-12


@pytest.mark.parametrize("n_ref", [1, 7, 8, 9, 1001, 65537])
def test_nn_far_queries_and_odd_sizes(n_ref):
    g = np.random.default_rng(n_ref)
    r = g.uniform(-20, 20, (n_ref, 3))
    far = g.normal(size=(5000, 3))
    far = far / np.linalg.norm(far, axis=1, keepdims=True) * g.uniform(100, 1000, (5000, 1))
    q = np.concatenate([far, g.uniform(-25, 25, (3001, 3))])
    _check_nn(q, r)


def _edge_cloud(g, n):
    cols = []
    for _ in range(3):
        e = M.voxel_edges([0.5, 0.2, 0.1][g.integers(0, 3)])
        cols.append(e[g.integers(0, e.shape[0], n)])
    p = np.stack(cols, 1)
    p[: n // 10, 0] = 50.0
    p[n // 10: n // 5, 1] = -50.0
    p[n // 5: n // 4, 2] = np.nextafter(50.0, 100.0)                    # just outside
    return np.concatenate([p, g.uniform(-60, 60, (n, 3)), _scan_like(200_000, 5)])


def _occupancy(pts, vs, counts=False):
    from lidiff_b200 import _lib
    h = _lib.get_handle("cuda")
    bins = M.voxel_bins(vs)
    e = torch.as_tensor(M.voxel_edges(vs), device="cuda")
    t = torch.as_tensor(pts, device="cuda")
    bits = torch.empty((bins ** 3 + 31) // 32, dtype=torch.int32, device="cuda")
    cnt = torch.empty(bins ** 3, dtype=torch.int32, device="cuda") if counts else None
    n_in = torch.zeros(1, dtype=torch.int64, device="cuda")
    h.voxel_occupancy(t, e, bits, cnt, n_in)
    occ = np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")[: bins ** 3].astype(bool)
    return occ, (cnt.cpu().numpy().view(np.uint32) if counts else None), int(n_in.item())


@pytest.mark.parametrize("vs", [0.5, 0.2])
def test_occupancy_and_counts_equal_histogramdd(vs):
    pts = _edge_cloud(np.random.default_rng(int(vs * 10)), 20_000)
    occ, cnt, n_in = _occupancy(pts, vs, counts=True)
    bins = M.voxel_bins(vs)
    ref = np.histogramdd(pts, bins=bins, range=[[-50, 50]] * 3)[0].reshape(-1)
    assert np.array_equal(cnt, ref.astype(np.uint32))
    assert np.array_equal(occ, ref > 0)
    assert n_in == int(ref.sum())


def test_occupancy_at_0_1_equals_sparse_restatement():
    pts = _edge_cloud(np.random.default_rng(3), 20_000)
    occ, _, n_in = _occupancy(pts, 0.1)
    e = M.voxel_edges(0.1)
    nb = e.shape[0] - 1
    b = np.searchsorted(e, pts, side="right") - 1
    b[pts == e[-1]] = nb - 1
    ok = ((b >= 0) & (b < nb)).all(1)
    cells = np.unique((b[ok, 0] * nb + b[ok, 1]) * nb + b[ok, 2])
    assert np.array_equal(np.nonzero(occ)[0], cells) and n_in == int(ok.sum())


def test_jsd_3d_and_bev_against_scipy():
    g = np.random.default_rng(4)
    gt = _scan_like(300_000, 7)
    pred = gt[g.choice(gt.shape[0], 150_000, replace=False)] + g.normal(0, 0.3, (150_000, 3))
    rec = M.evaluate_scan(gt, pred, thresholds=(), voxel_sizes=(), distances="none")
    rng = [[-50, 50]] * 3
    hg, hp = np.histogramdd(gt, bins=200, range=rng)[0], np.histogramdd(pred, bins=200, range=rng)[0]
    want3 = jensenshannon((hg / hg.sum()).ravel(), (hp / hp.sum()).ravel())
    bg, bp = np.clip(hg, 0, 1).sum(-1), np.clip(hp, 0, 1).sum(-1)
    wantb = jensenshannon((bg / bg.sum()).ravel(), (bp / bp.sum()).ravel())
    assert rec.jsd_3d == pytest.approx(want3, rel=1e-12)
    assert rec.jsd_bev == pytest.approx(wantb, rel=1e-12)


def test_against_the_reference_golden():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_metrics_goldens import metrics_pair
    ref = json.load(open(os.path.join(HERE, "golden", "metrics_reference.json")))
    gt, pred = metrics_pair(ref["seed"])
    assert (gt.shape[0], pred.shape[0]) == (ref["n_gt"], ref["n_pred"])
    rec = M.evaluate_scan(gt, pred, thresholds=np.linspace(*ref["pr_args"]), voxel_sizes=[0.5, 0.2, 0.1])
    iou = M.CompletionIoU([0.5, 0.2, 0.1])
    iou.add(rec)
    assert {str(k): [int(c) for c in iou.conf_matrix[i]] for i, k in enumerate(iou.voxel_sizes)} == ref["iou_conf"]
    assert {str(k): float(v) for k, v in iou.compute().items()} == ref["iou"]
    pr = M.PrecisionRecall(*ref["pr_args"])
    pr.add(rec)
    p, r, f = pr.compute_at_all_thresholds()
    assert (p, r) == (ref["precision"], ref["recall"])
    np.testing.assert_allclose(f, ref["f1"], rtol=1e-15)
    np.testing.assert_allclose(pr.compute_auc(), ref["auc"], rtol=1e-12)
    rm, cd = M.RMSE(), M.ChamferDistance()
    rm.add(rec)
    cd.add(rec)
    assert rm.compute()[0] == pytest.approx(ref["rmse"][0], rel=1e-12)
    assert cd.compute()[0] == pytest.approx(ref["chamfer"][0], rel=1e-12)
    assert rec.jsd_3d == pytest.approx(ref["jsd_3d"], rel=1e-12)
    assert rec.jsd_bev == pytest.approx(ref["jsd_bev"], rel=1e-12)


def test_two_evaluations_give_identical_bits():
    gt = _scan_like(400_000, 11)
    g = np.random.default_rng(5)
    pred = gt[g.choice(gt.shape[0], 250_000, replace=False)] + g.normal(0, 0.05, (250_000, 3))
    a, b = M.evaluate_scan(gt, pred), M.evaluate_scan(gt, pred)
    assert M.record_to_rows(a).numpy().tobytes() == M.record_to_rows(b).numpy().tobytes()
    d1, d2 = M.nn_distance(pred, gt), M.nn_distance(pred, gt)
    assert torch.equal(d1, d2)


def test_shim_point_cloud_distance_on_the_gpu():
    import lidiff_b200.shims as sh
    sh.install()
    import open3d as o3d
    g = np.random.default_rng(6)
    a, b = g.uniform(-30, 30, (50_000, 3)), _scan_like(120_000, 3)
    d = np.asarray(o3d.geometry.PointCloud(a).compute_point_cloud_distance(o3d.geometry.PointCloud(b)))
    assert np.abs(d - cKDTree(b).query(a)[0]).max() <= 1e-12


def _cli(args):
    from click.testing import CliRunner
    from lidiff_b200.tools.eval_path import main
    res = CliRunner().invoke(main, args, catch_exceptions=False)
    assert res.exit_code == 0, res.output
    return res.output


KEYS = {"jsd", "jsd_noclip_3d", "rmse_mean", "rmse_std", "ious", "cd_mean", "cd_std", "pr", "re", "f1"}


def test_eval_path_cli_ply_mode(tmp_path):
    from eval_sequence import make_sequence
    from lidiff_b200.tools import eval_path as E
    seq, pred_dir = make_sequence(str(tmp_path))
    out = _cli(["-p", pred_dir + "/", "--data", seq])
    assert out.count("JSD BEV:") == 4 and "FINAL RESULTS" in out
    res = json.load(open(os.path.join(pred_dir, "res_log.yaml")))
    assert set(res) == KEYS
    poses = E.load_poses(f"{seq}/calib.txt", f"{seq}/poses.txt")
    seq_map = np.load(f"{seq}/map_clean.npy")
    rm, cd, iou, pr = M.RMSE(), M.ChamferDistance(), M.CompletionIoU(), M.PrecisionRecall(*M.PR_ARGS)
    j3, jb = [], []
    for b, name in enumerate(sorted(os.listdir(f"{seq}/velodyne"))):
        pred, cur = E.scan_completion(seq, name, pred_dir, None, 50.0, "refine")
        gt = E.ground_truth(poses[b], cur, seq_map, 50.0)
        for acc in (rm, cd, iou, pr):
            acc.update(gt, pred)
        j3.append(M.compute_hist_metrics(gt, pred))
        jb.append(M.compute_hist_metrics(gt, pred, bev=True))
    want = {"jsd": float(np.mean(jb)), "jsd_noclip_3d": float(np.mean(j3)), "rmse_mean": float(rm.compute()[0]), "rmse_std": float(rm.compute()[1]),
            "ious": {str(k): float(v) for k, v in iou.compute().items()}, "cd_mean": float(cd.compute()[0]), "cd_std": float(cd.compute()[1]),
            "pr": float(pr.compute_auc()[0]), "re": float(pr.compute_auc()[1]), "f1": float(pr.compute_auc()[2])}
    assert res == want


def test_eval_path_cli_completion_mode(tmp_path):
    from eval_sequence import make_sequence
    seq, _ = make_sequence(str(tmp_path), beams=32, azimuths=1024)
    out_dir = tmp_path / "scored"
    out_dir.mkdir()
    _cli(["-p", str(out_dir) + "/", "--data", seq, "--random-weights", "-t", "1"])
    res = json.load(open(out_dir / "res_log.yaml"))
    assert set(res) == KEYS and set(res["ious"]) == {"0.5", "0.2", "0.1"}
    assert all(np.isfinite(v) for k, v in res.items() if k != "ious")
