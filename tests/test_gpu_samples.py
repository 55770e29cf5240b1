"""lb2_select_points / lb2_viewpoint_filter against their numpy restatements (tests/fake_samples_backend.py) and the open3d shim's
VoxelGrid, whole samples of lidiff_b200.datasets against the reference's recorded ones (tests/golden/samples_reference.npz), batch()
against collated items, and the test-mode CLI end to end."""
import os
import sys

import numpy as np
import pytest
import torch
import yaml
from click.testing import CliRunner

from fake_samples_backend import restate_select, restate_viewpoint
from lidiff_b200 import _lib
from lidiff_b200 import datasets as D

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_sample_goldens as G  # noqa: E402
from test_samples_host import assert_close_to_golden, make_set  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def select(points, labels, desc):
    h = _lib.get_handle(DEV)
    pts = torch.as_tensor(points).to(DEV).contiguous()
    lab = None if labels is None else torch.as_tensor(np.asarray(labels).view(np.int32)).to(DEV)
    out = torch.full((max(pts.shape[0], 1), 3), np.nan, dtype=torch.float64, device=DEV)
    cnt = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    h.select_points(pts, lab, desc, out, cnt, h.select_points_scratch(pts.shape[0]))
    return out[: int(cnt.item())].cpu().numpy()


def viewpoint(part, full, voxel=10.0):
    h = _lib.get_handle(DEV)
    p = torch.as_tensor(part, dtype=torch.float64).to(DEV).contiguous()
    f = torch.as_tensor(full, dtype=torch.float64).to(DEV).contiguous()
    out = torch.full((max(f.shape[0], 1), 3), np.nan, dtype=torch.float64, device=DEV)
    d_out = torch.full((2,), -1, dtype=torch.int32, device=DEV)
    h.viewpoint_filter(p, f, voxel, out, d_out, h.viewpoint_filter_scratch(p.shape[0], f.shape[0]))
    n, status = d_out.tolist()
    return out[:n].cpu().numpy(), status


def assert_rows(got, ref):
    """same rows in the same order; coordinates within 4 fp64 ulps of the row's magnitude (none differ where no transform is applied)"""
    assert got.shape == ref.shape, (got.shape, ref.shape)
    tol = 4 * np.spacing(np.abs(ref).sum(1, keepdims=True) + 1.0)
    assert (np.abs(got - ref) <= tol).all()


def random_rows(g, n, dtype, stride, scale=60.0):
    p = g.uniform(-scale, scale, (n, stride)).astype(dtype)
    p[g.choice(n, n // 50, replace=False), g.integers(0, 3, n // 50)] = np.nan
    p[g.choice(n, n // 50, replace=False), g.integers(0, 3, n // 50)] = np.inf
    p[g.choice(n, n // 50, replace=False), g.integers(0, 3, n // 50)] = -np.inf
    p[g.choice(n, n // 50, replace=False), :3] = 0.0
    return p


def labels_of(g, n):
    cls = g.choice([0, 1, 2, 9, 40, 251, 252, 253, 259, 0xFFFF], n)
    return (cls.astype(np.uint32) | (g.integers(0, 1 << 16, n).astype(np.uint32) << 16)).astype(np.uint32)


@pytest.mark.parametrize("dtype,stride", [(np.float32, 4), (np.float32, 3), (np.float64, 3), (np.float64, 4)])
def test_select_points_scan_and_map_crop(dtype, stride):
    g = np.random.default_rng(stride + (dtype == np.float64))
    p = random_rows(g, 100_003, dtype, stride)
    lab = labels_of(g, p.shape[0])
    pose = np.eye(4)
    a = 0.7
    pose[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
    pose[:3, 3] = [3.25, -7.5, 0.6]
    scan = D._desc(_lib.RANGE_FP32, r_min=3.5, r_max=50.0, z_min=-4.0)
    crop = D._desc(_lib.RANGE_FP64, center=pose[:3, 3], r_max=50.0, transform=np.linalg.inv(pose), z_min=-4.0)
    for labels, desc in ((lab, scan), (None, scan), (None, crop), (lab, crop), (None, D._desc())):
        ref = restate_select(p, labels, desc)
        assert ref.shape[0] > 1000
        assert_rows(select(p, labels, desc), ref)


def test_select_points_label_classes():
    """1 < (l & 0xFFFF) < 252 whatever the instance bits"""
    cls = np.arange(0, 1 << 16, dtype=np.uint32)
    lab = cls | (np.uint32(0xABCD) << 16)
    p = np.tile(np.array([[10.0, 0.0, 0.0, 0.0]], np.float32), (cls.shape[0], 1))
    p[:, 1] = np.arange(cls.shape[0], dtype=np.float32) * 1e-4
    got = select(p, lab, D._desc())
    kept = (cls > 1) & (cls < 252)
    np.testing.assert_array_equal(got, p[kept, :3].astype(np.float64))


def test_select_points_strict_range_boundaries():
    """r_min < d < r_max is strict, in fp32 for RANGE_FP32 and fp64 for RANGE_FP64; z > z_min is strict"""
    f32 = np.float32
    r = [f32(3.5), np.nextafter(f32(3.5), f32(0)), np.nextafter(f32(3.5), f32(9)), f32(50.0), np.nextafter(f32(50.0), f32(0)),
         np.nextafter(f32(50.0), f32(99))]
    p = np.zeros((len(r), 3), np.float32)
    p[:, 0] = r
    got = select(p, None, D._desc(_lib.RANGE_FP32, r_min=3.5, r_max=50.0))
    np.testing.assert_array_equal(got[:, 0], np.array([r[2], r[4]], np.float64))
    r64 = [3.5, np.nextafter(3.5, 0), np.nextafter(3.5, 9), 50.0, np.nextafter(50.0, 0), np.nextafter(50.0, 99)]
    q = np.zeros((len(r64), 3))
    q[:, 1] = r64
    got = select(q, None, D._desc(_lib.RANGE_FP64, r_min=3.5, r_max=50.0))
    np.testing.assert_array_equal(got[:, 1], [r64[2], r64[4]])
    # a value just below 50 in fp64 rounds to 50 in fp32: dropped by the fp32 range, kept by the fp64 one
    q = np.array([[0.0, 0.0, 50.0 - 1e-9]])
    assert select(q, None, D._desc(_lib.RANGE_FP32, r_max=50.0)).shape[0] == 0
    assert select(q, None, D._desc(_lib.RANGE_FP64, r_max=50.0)).shape[0] == 1
    z = np.array([[5.0, 0, -4.0], [5.0, 0, np.nextafter(-4.0, 0)], [5.0, 0, np.nextafter(-4.0, -9)]])
    np.testing.assert_array_equal(select(z, None, D._desc(z_min=-4.0)), z[1:2])


def test_select_points_non_finite_zero_and_empty():
    p = np.array([[np.nan, 5, 5], [5, np.inf, 5], [5, 5, -np.inf], [0, 0, 0], [6, 0, 0]], np.float32)
    np.testing.assert_array_equal(select(p, None, D._desc()), p[3:].astype(np.float64))
    np.testing.assert_array_equal(select(p, None, D._desc(_lib.RANGE_FP32, r_min=3.5, r_max=50)), p[4:].astype(np.float64))
    assert select(p, None, D._desc(_lib.RANGE_FP64, r_min=100.0, r_max=200.0)).shape == (0, 3)
    assert select(np.zeros((0, 3), np.float32), None, D._desc()).shape == (0, 3)


def test_select_points_order_across_many_blocks():
    """2^24 + 5 rows: every block's rows land after the earlier blocks' rows"""
    n = (1 << 24) + 5
    x = torch.arange(n, dtype=torch.float64, device=DEV)
    p = torch.stack([x, torch.zeros_like(x), torch.remainder(x * 7919, 13) - 6], 1).contiguous()
    h = _lib.get_handle(DEV)
    out = torch.empty((n, 3), dtype=torch.float64, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    h.select_points(p, None, D._desc(z_min=-4.0), out, cnt, h.select_points_scratch(n))
    keep = p[:, 2] > -4.0
    m = int(cnt.item())
    assert m == int(keep.sum())
    assert torch.equal(out[:m], p[keep])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_viewpoint_filter_matches_voxel_grid(seed):
    from lidiff_b200.shims.open3d.geometry import PointCloud, VoxelGrid
    g = np.random.default_rng(seed)
    part = g.uniform(-45, 25, (3000, 3)) * [1, 1, 0.1]
    full = g.uniform(-80, 60, (200_000, 3)) * [1, 1, 0.1]
    grid = VoxelGrid.create_from_point_cloud(PointCloud(part), 10.0)
    ref = full[np.asarray(grid.check_if_included(full))]
    got, status = viewpoint(part, full)
    assert status == 0
    np.testing.assert_array_equal(got, ref)
    keep, _ = restate_viewpoint(part, full, 10.0)
    np.testing.assert_array_equal(got, full[keep])


def test_viewpoint_filter_single_point_and_empty():
    from lidiff_b200.shims.open3d.geometry import PointCloud, VoxelGrid
    part = np.array([[-12.5, 3.0, -1.0]])
    full = np.concatenate([part + np.array([[dx, dy, dz]]) for dx in (-5.1, -4.9, 0, 4.9, 5.1) for dy in (-5.1, 0, 4.9, 5.1)
                           for dz in (-5.1, 0, 4.9)])
    grid = VoxelGrid.create_from_point_cloud(PointCloud(part), 10.0)
    got, status = viewpoint(part, full)
    np.testing.assert_array_equal(got, full[np.asarray(grid.check_if_included(full))])
    assert status == 0 and got.shape[0] == 3 * 2 * 2
    assert viewpoint(np.zeros((0, 3)), full)[0].shape == (0, 3)
    assert viewpoint(part, np.zeros((0, 3)))[0].shape == (0, 3)


@pytest.fixture(scope="module")
def data_root(tmp_path_factory):
    return G.make_dataset(str(tmp_path_factory.mktemp("kitti_gpu")))


@pytest.mark.parametrize("split", ["train", "validation", "test"])
def test_samples_match_reference(data_root, split):
    ds = make_set(data_root, split, device=DEV)
    np.random.seed(G.SEED)
    torch.manual_seed(G.SEED)
    for k, i in enumerate(G.RECORD[split]):
        item = ds[i]
        assert item[0].is_cuda and item[3].is_cuda
        assert_close_to_golden(split, k, item)


@pytest.mark.parametrize("indices", [[1], [4, 2], [0, 3, 1, 4]])
def test_batch_matches_collated_items(data_root, indices):
    ds = make_set(data_root, "train", device=DEV)
    np.random.seed(7)
    torch.manual_seed(7)
    ref = D.SparseSegmentCollation()([ds[i] for i in indices])
    np.random.seed(7)
    torch.manual_seed(7)
    b = ds.batch(indices)
    assert b["filename"] == ref["filename"]
    for key in ("pcd_full", "mean", "std", "pcd_part"):
        assert b[key].shape[0] == len(indices) and torch.equal(b[key], ref[key]), key


def test_cli_end_to_end(tmp_path):
    from lidiff_b200.tools import test_completion as TC
    root = str(tmp_path / "data")
    os.makedirs(os.path.join(root, "dataset", "sequences"))
    G.write_sequence(os.path.join(root, "dataset", "sequences", "08"), 2, 5)
    cfg = {"experiment": {"id": "t"}, "data": {"data_dir": root, "resolution": 0.05, "dataloader": "KITTI", "split": "train",
                                               "train": ["00"], "validation": ["08"], "num_points": 20000, "max_range": 50.0,
                                               "dataset_norm": False, "std_axis_norm": False},
           "train": {"uncond_w": 6.0, "batch_size": 2, "num_workers": 4},
           "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 50}}
    cfg_path = str(tmp_path / "config.yaml")
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)
    out = str(tmp_path / "out")
    args = ["-c", cfg_path, "--out", out, "--random-weights", "-T", "3"]
    r = CliRunner().invoke(TC.main, args, catch_exceptions=False)
    assert r.exit_code == 0, r.output
    plys = [os.path.join(out, "generated_pcd", "08", f"{k:06d}.ply") for k in range(2)]
    assert all(os.path.getsize(p) > 200 for p in plys)
    assert "CD Mean:" in r.output and "Precision:" in r.output and "F-Score:" in r.output
    r2 = CliRunner().invoke(TC.main, args, catch_exceptions=False)
    assert r2.exit_code == 0 and "Skipping generation" in r2.output and "CD Mean:" not in r2.output
