"""Import shims of SURVEY.md 8f-1: pytorch_lightning / natsort / open3d stand-ins the reference's inference script needs."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import lidiff_b200.shims as sh


@pytest.fixture(scope="module", autouse=True)
def _shims_on_path():
    sh.install()
    for m in ("open3d", "natsort", "pytorch_lightning"):          # a real install (none in this image) would be shadowed on purpose
        sys.modules.pop(m, None)
    yield


def test_natsorted_orders_numbers_naturally():
    from natsort import natsorted
    assert natsorted(["10.ply", "9.ply", "000100.ply", "1.ply", "a2", "a10"]) == ["1.ply", "9.ply", "10.ply", "000100.ply", "a2", "a10"]
    assert natsorted(["b3", "b20"], reverse=True) == ["b20", "b3"]


def test_lightning_module_hparams_device_and_partial_state_dict(tmp_path):
    from pytorch_lightning.core.lightning import LightningModule
    import yaml

    class M(LightningModule):
        def __init__(self, hp):
            super().__init__()
            self.save_hyperparameters(hp)
            self.lin = torch.nn.Linear(3, 2)

    m = M({"diff": {"t_steps": 1000}, "data": {"resolution": 0.05}})
    assert m.hparams["diff"]["t_steps"] == 1000 and m.device == torch.device("cpu")
    m.hparams["data"]["max_range"] = 50.0                                   # the reference mutates and dumps it (pipeline:49-56)
    assert yaml.safe_load(yaml.dump(m.hparams))["data"] == {"resolution": 0.05, "max_range": 50.0}
    sd = {"lin.weight": torch.ones(2, 3), "somebody.else": torch.zeros(1)}   # Lightning ckpt dicts hold all sub-models: strict=False
    res = m.load_state_dict(sd, strict=False)
    assert "lin.bias" in res.missing_keys and "somebody.else" in res.unexpected_keys and bool((m.lin.weight == 1).all())
    import pytorch_lightning as pl
    with pytest.raises(NotImplementedError):
        pl.Trainer(gpus=1)


def test_open3d_pointcloud_and_ply_round_trip(tmp_path):
    import open3d as o3d
    g = np.random.default_rng(0)
    pts = g.normal(size=(257, 3)) * [5, 5, 0.01]                               # a thin slab: normals ~ +-z
    pcd = o3d.geometry.PointCloud()
    pcd.points = o3d.utility.Vector3dVector(pts)
    assert np.array(pcd.points).shape == (257, 3) and not pcd.has_normals()
    for ascii_ in (False, True):
        f = str(tmp_path / f"a{int(ascii_)}.ply")
        o3d.io.write_point_cloud(f, pcd, write_ascii=ascii_)
        back = np.array(o3d.io.read_point_cloud(f).points)
        assert np.allclose(back, pts, rtol=0, atol=0 if not ascii_ else 1e-8)
    pcd.estimate_normals()
    n = np.asarray(pcd.normals)
    assert pcd.has_normals() and np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-5) and (np.abs(n[:, 2]) > 0.9).mean() > 0.9
    f = str(tmp_path / "n.ply")
    o3d.io.write_point_cloud(f, pcd)
    back = o3d.io.read_point_cloud(f)
    assert back.has_normals() and np.allclose(np.asarray(back.normals), n)
    with pytest.raises(RuntimeError):
        o3d.utility.Vector3dVector(np.zeros((4, 2)))
    from lidiff_b200.synth import read_ply_xyz                                   # the package's own reader agrees with the shim's writer
    assert np.allclose(read_ply_xyz(f), pts)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_open3d_fps_fails_loudly_without_gpu():
    import open3d as o3d
    pcd = o3d.geometry.PointCloud(np.zeros((10, 3)))
    with pytest.raises(RuntimeError):
        pcd.farthest_point_down_sample(3)


def reference_names():
    """what tests/golden/make_reference_goldens.py recorded from the reference (names, shapes, metric values)"""
    return json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_names.json")))


def test_reference_pipeline_script_imports_on_the_shims():
    """every name the reference's inference script binds from the shimmed packages (recorded when it was imported on the shims)
    resolves on the shims to an object of the same module and name; its DiffCompletion derives from the shim's LightningModule"""
    import importlib
    rec = reference_names()
    assert set(rec["pipeline_imports"]) == {"LightningModule", "ME", "natsorted", "o3d"}
    for gname, (src, qual) in rec["pipeline_imports"].items():
        m = importlib.import_module(src)
        obj = m if qual is None else getattr(m, qual)
        assert (obj.__name__ if qual is None else obj.__module__) == src, gname
    from pytorch_lightning.core.lightning import LightningModule
    assert rec["pipeline_base"] == [LightningModule.__module__ + "." + LightningModule.__qualname__]
    import open3d as o3d
    from natsort import natsorted
    import MinkowskiEngine as ME
    assert o3d.__version__.endswith("lidiff_b200.shim") and callable(natsorted) and ME.__name__ == "MinkowskiEngine"


def test_reference_metrics_module_runs_on_the_open3d_shim():
    """SURVEY 8f-4: the reference's lidiff/utils/metrics.py (RMSE, ChamferDistance, PrecisionRecall, CompletionIoU) ran unchanged on
    the open3d shim when tests/golden/reference_names.json was recorded; its results are restated here from the shim's
    nearest-neighbour distances (checked against scipy's exact k-d tree) and voxel grids, so a change of the shim shows"""
    from scipy.spatial import cKDTree
    import open3d as o3d
    rec = reference_names()["metrics"]
    g = np.random.default_rng(3)
    gt = g.normal(size=(6000, 3)) * [12, 12, 1.0]
    pred = gt[g.choice(6000, 4000, replace=False)] + g.normal(size=(4000, 3)) * 0.05
    pg, pp = o3d.geometry.PointCloud(gt), o3d.geometry.PointCloud(pred)
    d_pg = np.asarray(pp.compute_point_cloud_distance(pg))
    d_gp = np.asarray(pg.compute_point_cloud_distance(pp))
    assert np.allclose(d_pg, cKDTree(gt).query(pred)[0], rtol=0, atol=1e-9) and np.allclose(d_gp, cKDTree(pred).query(gt)[0], rtol=0, atol=1e-9)
    assert abs(rec["chamfer"] - 0.5 * (d_pg.mean() + d_gp.mean())) < 1e-12 and abs(rec["rmse"] - d_pg.mean()) < 1e-12
    p, r, f1 = rec["precision_recall_f1_at_0.1"]
    assert abs(p - 100.0 * (d_pg < 0.1).mean()) < 1e-9 and abs(r - 100.0 * (d_gp < 0.1).mean()) < 1e-9 and abs(f1 - 2 * p * r / (p + r)) < 1e-9
    assert all(0 <= v <= 100.000001 for v in rec["auc"])                  # percentages, normalised by the perfect predictor
    for vs, iou in rec["iou"].items():                                     # occupancy IoU of the two clouds' voxel grids
        grid = lambda x: {tuple(k) for k in np.floor(x / float(vs)).astype(np.int64)}
        a_, b_ = grid(gt), grid(pred)
        assert abs(iou - len(a_ & b_) / len(a_ | b_)) < 0.05, vs
    assert 0 < rec["iou"]["0.5"] <= rec["iou"]["1.0"] <= rec["iou"]["2.0"] <= 1
    # viewpoint mask of the training collation (collations.py:44-50): voxel-grid membership at 10 m
    grid = o3d.geometry.VoxelGrid.create_from_point_cloud(pp, voxel_size=10.0)
    inc = np.array(grid.check_if_included(o3d.utility.Vector3dVector(gt)))
    org = pred.min(0) - 5.0
    keys = {tuple(k) for k in np.floor((pred - org) / 10.0).astype(int)}
    assert np.array_equal(inc, np.array([tuple(k) in keys for k in np.floor((gt - org) / 10.0).astype(int)]))
