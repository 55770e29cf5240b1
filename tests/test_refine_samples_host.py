"""Host logic of lidiff_b200.datasets_refine and metrics.chamfer_distance on the numpy stand-in backend
(tests/fake_refine_backend.py): known answers of the kernels' restatements, the reference's recorded samples for the train,
validation and test loaders (tests/golden/refine_samples_reference.npz), the window rule, the errors, the collation and the data
module's splits, pytorch3d's Chamfer op sequence, and the reference's refinement modules importing unchanged on the shims."""
import importlib
import os
import shutil
import sys
import types

import numpy as np
import pytest
import torch
from torch.utils.data import RandomSampler, SequentialSampler

import fake_refine_backend as F
from lidiff_b200 import datasets_refine as R
from lidiff_b200 import metrics
from lidiff_b200.kitti import load_poses

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_refine_sample_goldens as G  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "refine_samples_reference.npz"))


@pytest.fixture(scope="module")
def data_root(tmp_path_factory):
    return G.make_dataset(str(tmp_path_factory.mktemp("kitti")))


@pytest.fixture
def fake(monkeypatch):
    return F.install(monkeypatch)


def make_set(root, split, device="cpu"):
    return R.TemporalKITTISet(root, G.SCAN_WINDOW, G.split_seqs(split), G.split_name(split), G.RESOLUTION, G.NUM_POINTS, "refine",
                              device=device)


def assert_close_to_golden(split, k, item):
    """rows in the same order: within 2 float32 ulps of the golden (1 ulp before the scale in [0.95, 1.05]) for the augmented train
    split, equal otherwise (fp64 arithmetic in numpy's order); mean / std within 1e-12 relative"""
    p_full, mean, std, p_noise, window = item
    for name, got in (("pcd_full", p_full), ("pcd_noise", p_noise)):
        ref = GOLDEN[G.record_key(split, k, name)]
        got = got.cpu().numpy()
        assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape, got.dtype, ref.dtype)
        if split == "train":
            err = np.abs(got - ref)
            assert (err <= 2 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)).all(), (split, k, name, err.max())
        else:
            np.testing.assert_array_equal(got, ref, err_msg=f"{split} {k} {name}")
    for name, got in (("mean", mean), ("std", std)):
        np.testing.assert_allclose(got.cpu().numpy(), GOLDEN[G.record_key(split, k, name)], rtol=1e-12, atol=0,
                                   err_msg=f"{split} {k} {name}")
    assert ["/".join(p.split("/")[-3:]) for p in window] == list(GOLDEN[G.record_key(split, k, "window")])


# ---- known answers of the restatements ------------------------------------------------------------------------------------------
def _identity12():
    return np.eye(4)[:3].reshape(-1)


def test_aggregate_label_rule_keeps_classes_0_and_1():
    pts = np.tile(np.array([[5.0, 0.0, 0.0, 0.5]], np.float32), (6, 1))
    lab = np.array([0, 1, 251, 252, (7 << 16) | 251, (7 << 16) | 252], np.uint32)
    w, n_before = F.restate_aggregate(pts, lab, [0], [_identity12()], _identity12(), 6)
    assert w.shape == (4, 3) and n_before == 4


def test_aggregate_keeps_inf_and_drops_nan_and_near_rows():
    pts = np.array([[np.inf, 1, 1, 0], [np.nan, 1, 1, 0], [3.4, 0, 0, 9], [3.6, 0, 0, 0], [-np.inf, 0, 0, 0]], np.float32)
    w, _ = F.restate_aggregate(pts, np.full(5, 40, np.uint32), [0], [_identity12()], _identity12(), 5)
    assert w.shape == (3, 3)                       # 3.4 m stays out although remission would lift the map path's range
    # the infinite rows survive as non-finite rows (inf * 0 = NaN in the pose products) for the later stages to drop
    assert not np.isfinite(w[0]).all() and w[1, 0] == np.float64(np.float32(3.6)) and not np.isfinite(w[2]).all()


def test_aggregate_splits_at_the_frame_scan_and_applies_both_poses():
    pts = np.array([[10, 0, 0, 0], [0, 10, 0, 0], [0, 0, 10, 0], [1, 1, 1, 0]], np.float32)
    shift = lambda t: np.array([[1, 0, 0, t], [0, 1, 0, 0], [0, 0, 1, 0]], np.float64).reshape(-1)
    w, n_before = F.restate_aggregate(pts, np.full(4, 9, np.uint32), [0, 2], [shift(1.0), shift(2.0)], shift(-5.0), 2)
    assert n_before == 2 and w.shape == (3, 3)     # the 1.7 m row of the frame scan is dropped
    np.testing.assert_array_equal(w[:, 0], [10 + 1 - 5, 0 + 1 - 5, 0 + 2 - 5])


def test_voxel_first_floors_negative_coordinates_and_keeps_first_rows_in_order():
    p = np.array([[0.31, 0, 0], [-0.05, 0, 0], [0.35, 0, 0], [-0.01, 0, 0], [0.05, 0, 0], [np.nan, 0, 0], [np.inf, 0, 0],
                  [60.0, 0, 0], [60.01, 0, 0]])
    w, status = F.restate_voxel_first(p, 0.1, 50.0)
    assert status == 0
    np.testing.assert_array_equal(w[:, 0], [0.31, -0.05, 0.05])        # 60 m wins its voxel, then fails the range test
    w, status = F.restate_voxel_first(np.array([[2e5, 0, 0], [1.0, 0, 0]]), 0.1, 50.0)
    assert status == 1 and w.shape == (1, 3)


def test_jitter_clips_the_scaled_draw():
    p = np.zeros((3, 3))
    r = np.array([[1.0, -1.0, 0.5], [3.0, -3.0, 0.0], [0.0, 0.0, 0.0]])
    w = F.restate_jitter(p + [[49.9, 0, 0], [0, 0, 0], [50.0, 0, 0]], r, 0.2, 0.3, 50.0)
    np.testing.assert_array_equal(w, [[0.3, -0.3, 0.0]])          # 50.1 m and exactly 50 m fail the range test


# ---- the dataset ------------------------------------------------------------------------------------------------------------
def test_window_rule():
    names = [f"{i:06d}.bin" for i in range(7)]
    assert R.window_list(names, 3) == [names[0:3], names[1:4], names[2:5], names[3:7]]
    assert R.window_list(names[:1], 3) == [names[:1]]
    assert R.window_list(names[:4], 3) == [names[:4]]
    assert R.window_list([], 3) == []
    assert [len(w) for w in R.window_list(names, 1)] == [1] * 7


def test_aggregate_undoes_with_the_last_scan_of_the_window(data_root, fake):
    ds = make_set(data_root, "validation")
    window = ds.points_datapath[0]
    assert len(window) == 4
    seq = os.path.dirname(os.path.dirname(window[0]))
    poses = load_poses(os.path.join(seq, "calib.txt"), os.path.join(seq, "poses.txt"))
    undo = np.linalg.inv(poses[3])[:3].reshape(-1)
    parts = []
    for k in (0, 1, 3, 2):                           # the frame scan len // 2 = 2 last
        p = np.fromfile(window[k], np.float32).reshape(-1, 4)
        lab = np.fromfile(window[k].replace("velodyne", "labels").replace(".bin", ".label"), np.uint32)
        parts.append(F.restate_aggregate(p, lab, [0], [poses[k][:3].reshape(-1)], undo, p.shape[0])[0])
    np.testing.assert_array_equal(ds.aggregate(0).numpy(), np.concatenate(parts))


@pytest.mark.parametrize("split", ["train", "validation", "test"])
def test_samples_match_the_reference(data_root, fake, split):
    ds = make_set(data_root, split)
    np.random.seed(G.SEED)
    torch.manual_seed(G.SEED)
    for k, i in enumerate(G.RECORD[split]):
        assert int(GOLDEN[G.record_key(split, k, "index")]) == i
        assert_close_to_golden(split, k, ds[i])


def test_samples_cover_repeat_and_truncation():
    full = [len(np.unique(GOLDEN[G.record_key(s, k, "pcd_full")], axis=0)) for s in G.RECORD for k in range(len(G.RECORD[s]))]
    noise = [len(np.unique(GOLDEN[G.record_key(s, k, "pcd_noise")], axis=0)) for s in G.RECORD for k in range(len(G.RECORD[s]))]
    assert min(full) < 2 * G.NUM_POINTS and max(full) == 2 * G.NUM_POINTS
    assert min(noise) < G.NUM_POINTS and max(noise) == G.NUM_POINTS


def test_random_draw_order(data_root, fake, monkeypatch):
    """numpy's randn over every aggregated row, then torch's randperm of the ground truth, then of the noisy rows"""
    calls = []
    randn, randperm = np.random.randn, torch.randperm
    monkeypatch.setattr(np.random, "randn", lambda *s: calls.append(("randn", s)) or randn(*s))
    monkeypatch.setattr(torch, "randperm", lambda n, **kw: calls.append(("randperm", n)) or randperm(n, **kw))
    ds = make_set(data_root, "validation")
    n = ds.aggregate(0).shape[0]
    ds[0]
    assert [c[0] for c in calls] == ["randn", "randperm", "randperm"] and calls[0][1] == (1, n, 3)


def _one_scan_root(tmp_path, data_root, edit):
    root = str(tmp_path / "kitti")
    shutil.copytree(os.path.join(data_root, "dataset", "sequences", "01"), os.path.join(root, "dataset", "sequences", "01"))
    edit(os.path.join(root, "dataset", "sequences", "01"))
    return R.TemporalKITTISet(root, 3, ["01"], "validation", 0.05, 100, "refine", device="cpu")


def test_errors_name_the_window(tmp_path, data_root, fake):
    def all_moving(seq):
        p = os.path.join(seq, "labels", "000000.label")
        np.full(os.path.getsize(p) // 4, 252, np.uint32).tofile(p)
    with pytest.raises(ValueError, match="000000.bin .* frame scan"):
        _one_scan_root(tmp_path / "a", data_root, all_moving)[0]

    def far(seq):
        np.tile(np.array([[60.0, 0, 0, 0.5]], np.float32), (10, 1)).tofile(os.path.join(seq, "velodyne", "000000.bin"))
        np.full(10, 40, np.uint32).tofile(os.path.join(seq, "labels", "000000.label"))
    with pytest.raises(ValueError, match="000000.bin .* within 50 m"):
        _one_scan_root(tmp_path / "b", data_root, far)[0]
    with pytest.raises(ValueError, match="label file"):
        _one_scan_root(tmp_path / "c", data_root, lambda seq: os.remove(os.path.join(seq, "labels", "000000.label")))[0]

    def renamed(seq):
        os.rename(os.path.join(seq, "velodyne", "000000.bin"), os.path.join(seq, "velodyne", "scan_a.bin"))
        os.rename(os.path.join(seq, "labels", "000000.label"), os.path.join(seq, "labels", "scan_a.label"))
    with pytest.raises(ValueError, match="integer stem"):
        _one_scan_root(tmp_path / "d", data_root, renamed)[0]


def test_collation_keys_and_shapes(data_root, fake):
    ds = make_set(data_root, "validation")
    b = ds.batch([0])
    assert set(b) == {"pcd_full", "mean", "std", "pcd_noise", "filename"}
    assert b["pcd_full"].shape == (1, 2 * G.NUM_POINTS, 3) and b["pcd_noise"].shape == (1, G.NUM_POINTS, 3)
    assert b["pcd_full"].dtype == torch.float32 and len(b["filename"]) == 1 and len(b["filename"][0]) == 4


def test_data_module_splits(data_root, fake):
    cfg = {"data": {"data_dir": data_root, "resolution": 0.05, "split": "train", "train": ["00", "01"], "validation": ["08"],
                    "scan_window": 3, "num_points": 100},
           "train": {"batch_size": 2, "num_workers": 4, "mode": "refine"}}
    dm = R.dataloaders["KITTI"](cfg, device="cpu")
    tr, va, te = dm.train_dataloader(), dm.val_dataloader(), dm.test_dataloader()
    assert isinstance(tr.sampler, RandomSampler) and tr.batch_size == 2 and tr.dataset.split == "train"
    assert isinstance(va.sampler, SequentialSampler) and va.batch_size == 1 and va.dataset.seqs == ["08"]
    assert te.batch_size == 1 and te.dataset.seqs == ["00", "01"] and te.dataset.split == "validation"
    assert len(te.dataset) == 5 and len(va.dataset) == 1


# ---- Chamfer distance -------------------------------------------------------------------------------------------------------
def _p3d_reference(x, y):
    """pytorch3d 0.7.1's chamfer_distance op sequence over an fp64 brute-force argmin (lowest index on ties)"""
    def d2(q, r):
        j = ((q.double()[:, None] - r.double()[None]) ** 2).sum(-1).argmin(1)
        return ((q - r[j]) ** 2).sum(-1)
    cx = torch.stack([d2(x[b], y[b]) for b in range(x.shape[0])]).sum(1)
    cy = torch.stack([d2(y[b], x[b]) for b in range(x.shape[0])]).sum(1)
    cx /= torch.full((x.shape[0],), x.shape[1]).clamp(min=1)
    cy /= torch.full((x.shape[0],), y.shape[1]).clamp(min=1)
    cx, cy = cx.sum(), cy.sum()
    cx /= x.shape[0]
    cy /= x.shape[0]
    return cx + cy


def test_chamfer_op_sequence(fake):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 50, 3, generator=g)
    y = torch.cat([torch.randn(2, 30, 3, generator=g), x[:, :5]], 1)        # exact duplicates: zero distances
    loss, normals = metrics.chamfer_distance(x, y)
    assert normals is None and loss.dtype == torch.float32 and loss.shape == ()
    assert loss.item() == _p3d_reference(x, y).item()


def test_chamfer_ties_take_the_lowest_index(fake):
    x = torch.tensor([[[0.0, 0.0, 0.0]]])
    y = torch.tensor([[[1.0, 0.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 2.0, 0.0]]])
    loss, _ = metrics.chamfer_distance(x, y)
    assert loss.item() == 1.0 + (1.0 + 1.0 + 4.0) / 3


@pytest.mark.parametrize("kw", [{"x_lengths": torch.tensor([2])}, {"y_normals": torch.zeros(1, 2, 3)}, {"weights": torch.ones(1)},
                                {"batch_reduction": "sum"}, {"point_reduction": None}, {"norm": 1}])
def test_chamfer_non_default_arguments_raise(fake, kw):
    with pytest.raises(NotImplementedError):
        metrics.chamfer_distance(torch.zeros(1, 2, 3), torch.zeros(1, 2, 3), **kw)


# ---- the reference's modules on the shims ---------------------------------------------------------------------------------
REF = os.environ.get("LIDIFF_REFERENCE_DIR", "")


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "lidiff")), reason="LIDIFF_REFERENCE_DIR (a reference checkout) is not set")
def test_reference_refine_modules_import_unchanged_on_the_shims(monkeypatch):
    import lidiff_b200.shims as sh
    sh.install()
    for m in ("pytorch_lightning", "pytorch3d", "pytorch3d.loss"):
        sys.modules.pop(m, None)
    monkeypatch.setitem(sys.modules, "hdbscan", types.ModuleType("hdbscan"))
    mpl, plt = types.ModuleType("matplotlib"), types.ModuleType("matplotlib.pyplot")
    mpl.pyplot = plt
    monkeypatch.setitem(sys.modules, "matplotlib", mpl)
    monkeypatch.setitem(sys.modules, "matplotlib.pyplot", plt)
    monkeypatch.syspath_prepend(REF)
    for k in [k for k in sys.modules if k == "lidiff" or k.startswith("lidiff.")]:
        monkeypatch.delitem(sys.modules, k)
    models = importlib.import_module("lidiff.models.models_refine")
    data = importlib.import_module("lidiff.datasets.datasets_refine")
    from pytorch_lightning import LightningDataModule
    assert models.chamfer_distance is metrics.chamfer_distance
    assert issubclass(data.TemporalKittiDataModule, LightningDataModule)
