"""Host logic of lidiff_b200.metrics and the eval_path CLI on the CPU stand-in backend (tests/fake_metrics_backend.py): calib / pose
parsing, the ground-truth crop, `.ply` scoring, the scan-order fold of per-scan records, and the reference's metric semantics
restated with scipy / numpy."""
import json
import random

import numpy as np
import pytest
import scipy.integrate
from scipy.spatial import cKDTree
from scipy.spatial.distance import jensenshannon

import fake_metrics_backend
from eval_sequence import lidar_pose, make_sequence
from lidiff_b200 import metrics as M
from lidiff_b200.tools import eval_path as E


@pytest.fixture
def fake(monkeypatch):
    return fake_metrics_backend.install(monkeypatch)


@pytest.fixture(scope="module")
def sequence(tmp_path_factory):
    return make_sequence(str(tmp_path_factory.mktemp("eval_seq")))


def test_calib_and_poses_give_lidar_frame_poses(sequence):
    seq, _ = sequence
    poses = E.load_poses(f"{seq}/calib.txt", f"{seq}/poses.txt")
    assert len(poses) == 3
    for b, p in enumerate(poses):
        np.testing.assert_allclose(p, lidar_pose(b), atol=1e-9)


def test_ground_truth_crop_keeps_the_scans_own_points(sequence):
    seq, _ = sequence
    poses = E.load_poses(f"{seq}/calib.txt", f"{seq}/poses.txt")
    seq_map = np.load(f"{seq}/map_clean.npy")
    for b in range(3):
        raw = np.fromfile(f"{seq}/velodyne/{b:06d}.bin", dtype=np.float32).reshape(-1, 4)
        cur = raw[np.sqrt((raw[:, :3] ** 2).sum(1)) < 50.0, :3]
        gt = E.ground_truth(poses[b], cur, seq_map, 50.0)
        assert gt.shape[0] > cur.shape[0] // 2
        assert ((gt[:, 2] > -4.0) & (gt[:, 2] < 4.4)).all()
        assert (np.sqrt((gt ** 2).sum(1)) < 50.0 + 1e-6).all()           # the crop is around the pose: within range in the scan frame
        # every map point inside the range, the z band and the scan's own 10 m voxels is kept
        world = seq_map @ np.linalg.inv(poses[b])[:3, :3].T + np.linalg.inv(poses[b])[:3, 3]
        lo = cur.astype(np.float64).min(0) - 5.0
        occupied = {tuple(v) for v in np.floor((cur.astype(np.float64) - lo) / 10.0).astype(np.int64)}
        d = np.sqrt(((seq_map - poses[b][:3, 3]) ** 2).sum(1))
        keep = (d < 50.0) & (world[:, 2] > -4.0) & (world[:, 2] < 4.4)
        keep &= np.array([tuple(v) in occupied for v in np.floor((world - lo) / 10.0).astype(np.int64)])
        assert gt.shape[0] == int(keep.sum())


def _restated(gt, pred):
    """the reference's per-scan metrics restated with scipy / numpy (0.1 m IoU: sparse cells, not a dense 1000^3 grid)"""
    d_pg, _ = cKDTree(gt).query(pred)
    d_gp, _ = cKDTree(pred).query(gt)
    out = {"rmse": d_pg.mean(), "cd": (d_gp.mean() + d_pg.mean()) / 2}
    thr = np.linspace(*M.PR_ARGS)
    p = np.array([100 / len(d_pg) * (d_pg < t).sum() for t in thr])
    r = np.array([100 / len(d_gp) * (d_gp < t).sum() for t in thr])
    f = np.where((p == 0) | (r == 0), 0, 2 * p * r / np.where(p + r == 0, 1, p + r))
    out["pr"], out["re"], out["f1"] = p, r, f
    cells = {}
    for vs in M.VOXEL_SIZES:
        e = M.voxel_edges(vs)
        nb = e.shape[0] - 1

        def occ(x):
            b = np.searchsorted(e, x, side="right") - 1
            b[x == e[-1]] = nb - 1
            ok = ((b >= 0) & (b < nb)).all(1)
            return set(((b[ok, 0] * nb + b[ok, 1]) * nb + b[ok, 2]).tolist())
        a, c = occ(gt), occ(pred)
        cells[vs] = (len(a & c), len(a - c), len(c - a))
    out["conf"] = cells
    rng = [[-50, 50]] * 3
    hg, hp = np.histogramdd(gt, bins=200, range=rng)[0], np.histogramdd(pred, bins=200, range=rng)[0]
    out["jsd_3d"] = jensenshannon((hg / hg.sum()).ravel(), (hp / hp.sum()).ravel())
    bg, bp = np.clip(hg, 0, 1).sum(-1), np.clip(hp, 0, 1).sum(-1)
    out["jsd_bev"] = jensenshannon((bg / bg.sum()).ravel(), (bp / bp.sum()).ravel())
    return out


def _clouds(sequence):
    seq, pred_dir = sequence
    poses = E.load_poses(f"{seq}/calib.txt", f"{seq}/poses.txt")
    seq_map = np.load(f"{seq}/map_clean.npy")
    out = []
    for b, name in enumerate(E.natural_sorted(__import__("os").listdir(f"{seq}/velodyne"))):
        pred, cur = E.scan_completion(seq, name, pred_dir, None, 50.0, "refine")
        out.append((E.ground_truth(poses[b], cur, seq_map, 50.0), pred))
    return out


def test_ply_mode_res_log_matches_the_restated_reference(fake, sequence, capsys):
    seq, pred_dir = sequence
    n, local = E.score_scans(seq, pred_dir, None, 50.0, "refine", "cpu")
    assert n == 3 and sorted(local) == [0, 1, 2]
    res = E.fold({b: M.record_from_rows(r) for b, r in local.items()})
    printed = capsys.readouterr().out
    assert printed.count("JSD 3D:") == 3 and printed.count("Voxel 0.1cm IOU:") == 3
    ref = [_restated(gt, pred) for gt, pred in _clouds(sequence)]
    rmse = np.array([r["rmse"] for r in ref])
    cd = np.array([r["cd"] for r in ref])
    assert res["rmse_mean"] == pytest.approx(rmse.mean(), rel=1e-12) and res["rmse_std"] == pytest.approx(rmse.std(), rel=1e-9)
    assert res["cd_mean"] == pytest.approx(cd.mean(), rel=1e-12) and res["cd_std"] == pytest.approx(cd.std(), rel=1e-9)
    thr = np.linspace(*M.PR_ARGS)
    dx = thr[1] - thr[0]
    perfect = scipy.integrate.simpson(np.ones_like(thr), dx=dx)
    for key in ("pr", "re", "f1"):
        curve = np.mean([r[key] for r in ref], axis=0)
        assert res[key] == pytest.approx(scipy.integrate.simpson(curve, dx=dx) / perfect, rel=1e-12)
    for vs in M.VOXEL_SIZES:
        tp, fn, fp = (sum(r["conf"][vs][i] for r in ref) for i in range(3))
        assert res["ious"][vs] == tp / (tp + fn + fp + 1e-15)
    assert res["jsd_noclip_3d"] == pytest.approx(np.mean([r["jsd_3d"] for r in ref]), rel=1e-12)
    assert res["jsd"] == pytest.approx(np.mean([r["jsd_bev"] for r in ref]), rel=1e-12)
    assert set(json.loads(json.dumps(E.to_json(res)))) == {"jsd", "jsd_noclip_3d", "rmse_mean", "rmse_std", "ious", "cd_mean", "cd_std",
                                                           "pr", "re", "f1"}


def test_fold_does_not_depend_on_the_rank_split(fake, sequence):
    seq, pred_dir = sequence
    _, one = E.score_scans(seq, pred_dir, None, 50.0, "refine", "cpu")
    split = {}
    for rank in (1, 0):
        split.update(E.score_scans(seq, pred_dir, None, 50.0, "refine", "cpu", rank=rank, world=2)[1])
    keys = list(split)
    random.Random(0).shuffle(keys)
    shuffled = {b: split[b] for b in keys}
    a = E.to_json(E.fold({b: M.record_from_rows(r) for b, r in one.items()}, verbose=False))
    b = E.to_json(E.fold({b: M.record_from_rows(r) for b, r in shuffled.items()}, verbose=False))
    assert json.dumps(a) == json.dumps(b)


def test_record_rows_round_trip_is_exact(fake, sequence):
    gt, pred = _clouds(sequence)[0]
    rec = M.evaluate_scan(gt, pred)
    back = M.record_from_rows(M.record_to_rows(rec))
    for f in ("n_gt", "n_pred", "sum_pred_to_gt", "sum_gt_to_pred", "jsd_3d", "jsd_bev", "voxel_sizes"):
        assert getattr(back, f) == getattr(rec, f), f
    for f in ("thresholds", "cnt_pred_to_gt", "cnt_gt_to_pred", "conf"):
        assert np.array_equal(getattr(back, f), getattr(rec, f)) and getattr(back, f).dtype == getattr(rec, f).dtype, f


def test_accumulators_match_one_evaluation(fake, sequence):
    gt, pred = _clouds(sequence)[1]
    rec = M.evaluate_scan(gt, pred)
    for cls, args in ((M.RMSE, ()), (M.ChamferDistance, ()), (M.CompletionIoU, ()), (M.PrecisionRecall, M.PR_ARGS)):
        a, b = cls(*args), cls(*args)
        a.update(gt, pred)
        b.add(rec)
        if cls is M.PrecisionRecall:
            assert a.compute_at_all_thresholds() == b.compute_at_all_thresholds()
            assert a.compute_at_threshold(0.07) == b.compute_at_threshold(0.07)
        else:
            assert a.compute() == b.compute()
    assert M.compute_hist_metrics(gt, pred, bev=True) == rec.jsd_bev
    assert M.compute_hist_metrics(gt, pred) == rec.jsd_3d


def test_empty_or_out_of_range_clouds_raise(fake):
    inside = np.random.default_rng(0).uniform(-10, 10, (100, 3))
    with pytest.raises(ValueError):
        M.evaluate_scan(inside, np.zeros((0, 3)))
    with pytest.raises(ValueError):
        M.evaluate_scan(inside, inside + 200.0)
    with pytest.raises(ValueError):
        M.compute_hist_metrics(inside + 200.0, inside)
