"""lb2_aggregate_window / lb2_jitter_filter / lb2_voxel_first_f64 against their numpy restatements (tests/fake_refine_backend.py),
whole samples of lidiff_b200.datasets_refine against the reference's recorded ones (tests/golden/refine_samples_reference.npz),
metrics.chamfer_distance against brute force and scipy's k-d tree, and the refinement test-mode CLI end to end."""
import os
import sys

import numpy as np
import pytest
import torch
import yaml
from click.testing import CliRunner

import fake_refine_backend as F
from lidiff_b200 import _lib, metrics
from lidiff_b200 import datasets_refine as R

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_refine_sample_goldens as G  # noqa: E402
from test_refine_samples_host import assert_close_to_golden  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def aggregate(points, labels, starts, poses, undo12, split):
    h = _lib.get_handle(DEV)
    n = points.shape[0]
    seg = np.zeros(len(starts), R.SEGMENT_DTYPE)
    seg["start"], seg["m"] = starts, np.asarray(poses).reshape(-1, 12)
    out = torch.full((max(n, 1), 3), np.nan, dtype=torch.float64, device=DEV)
    d_out = torch.full((2,), -1, dtype=torch.int32, device=DEV)
    h.aggregate_window(torch.from_numpy(points).to(DEV), torch.from_numpy(labels.view(np.int32)).to(DEV),
                       torch.from_numpy(seg.view(np.uint8)).to(DEV), len(starts), undo12, split, out, d_out, h.aggregate_window_scratch(n))
    m, before = d_out.tolist()
    return out[:m].cpu().numpy(), before


def jitter(p, r):
    h = _lib.get_handle(DEV)
    pt, rt = torch.from_numpy(p).to(DEV), torch.from_numpy(r).to(DEV)
    out = torch.full((max(p.shape[0], 1), 3), np.nan, dtype=torch.float64, device=DEV)
    cnt = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    h.jitter_filter(pt, rt, 0.2, 0.3, 50.0, out, cnt, h.jitter_filter_scratch(p.shape[0]))
    return out[: int(cnt.item())].cpu().numpy()


def voxel_first(p):
    h = _lib.get_handle(DEV)
    pt = torch.from_numpy(p).to(DEV)
    out = torch.full((max(p.shape[0], 1), 3), np.nan, dtype=torch.float64, device=DEV)
    d_out = torch.full((2,), -1, dtype=torch.int32, device=DEV)
    h.voxel_first_f64(pt, 0.1, 50.0, out, d_out, h.voxel_first_f64_scratch(p.shape[0]))
    n, status = d_out.tolist()
    return out[:n].cpu().numpy(), status


def random_window(g, sizes, scale=60.0):
    """scans of `sizes` rows with non-finite coordinates, label edges, rows at the origin and an all-filtered scan when a size is
    negative (its rows are all label 252)"""
    rows, labs = [], []
    for s in sizes:
        k = abs(s)
        p = g.uniform(-scale, scale, (k, 4)).astype(np.float32)
        if k >= 50:
            for v in (np.nan, np.inf, -np.inf):
                p[g.choice(k, k // 50, replace=False), g.integers(0, 3, k // 50)] = v
            p[g.choice(k, k // 50, replace=False), :3] = 0.0
        cls = g.choice([0, 1, 2, 40, 251, 252, 253, 0xFFFF], k) if s > 0 else np.full(k, 252)
        labs.append((cls.astype(np.uint32) | (g.integers(0, 1 << 16, k).astype(np.uint32) << 16)).astype(np.uint32))
        rows.append(p)
    starts = np.cumsum([0] + [abs(s) for s in sizes[:-1]])
    poses = []
    for b in range(len(sizes)):
        a = 0.3 * b + 0.1
        poses.append(np.array([[np.cos(a), -np.sin(a), 0.01, 1.7 * b], [np.sin(a), np.cos(a), -0.02, 0.3 * b], [0.02, 0.01, 1.0, 0.05]]))
    undo = np.linalg.inv(np.vstack([poses[-1], [0, 0, 0, 1]]))[:3].reshape(-1)
    return np.concatenate(rows), np.concatenate(labs), starts, np.stack(poses), undo


@pytest.mark.parametrize("sizes", [[5000], [3000, 0, 7000, 4500], [2048, -900, 1, 2049], [20000, -3000]])
def test_aggregate_window_matches_restatement(sizes):
    g = np.random.default_rng(len(sizes) + sum(abs(s) for s in sizes))
    pts, lab, starts, poses, undo = random_window(g, sizes)
    split = int(starts[-1])
    got, before = aggregate(pts, lab, starts, poses, undo, split)
    ref, ref_before = F.restate_aggregate(pts, lab, starts, poses, undo, split)
    assert before == ref_before and got.shape == ref.shape
    np.testing.assert_array_equal(got, ref)          # elementwise fp64 in a fixed order: the same bits, NaN in the same places


def test_aggregate_window_above_the_unique_build_limit():
    """a 4.5 M-row window (more than lb2_unique_build's 4 194 304 rows) with empty and all-filtered scans"""
    g = np.random.default_rng(45)
    sizes = [150_000] * 29 + [0, -100_000] + [150_000] * 1
    pts, lab, starts, poses, undo = random_window(g, sizes)
    assert pts.shape[0] > 4_194_304
    got, before = aggregate(pts, lab, starts, poses, undo, int(starts[-1]))
    ref, ref_before = F.restate_aggregate(pts, lab, starts, poses, undo, int(starts[-1]))
    assert before == ref_before
    np.testing.assert_array_equal(got, ref)
    r = g.standard_normal(got.shape)
    np.testing.assert_array_equal(jitter(got, r), F.restate_jitter(got, r, 0.2, 0.3, 50.0))
    v, status = voxel_first(got)
    rv, rstatus = F.restate_voxel_first(got, 0.1, 50.0)
    assert status == rstatus == 0
    np.testing.assert_array_equal(v, rv)


@pytest.mark.parametrize("n", [1, 777, 2048, 100_000])
def test_jitter_filter_matches_restatement(n):
    g = np.random.default_rng(n)
    p = g.uniform(-55, 55, (n, 3))
    if n > 100:
        p[g.choice(n, n // 50, replace=False), g.integers(0, 3, n // 50)] = np.nan
        p[g.choice(n, n // 50, replace=False), g.integers(0, 3, n // 50)] = np.inf
    r = g.standard_normal((n, 3)) * 2.0                   # many draws beyond the clip
    np.testing.assert_array_equal(jitter(p, r), F.restate_jitter(p, r, 0.2, 0.3, 50.0))


@pytest.mark.parametrize("case", ["random", "duplicates", "negative", "nonfinite"])
def test_voxel_first_matches_restatement(case):
    g = np.random.default_rng(len(case))
    n = 300_000
    if case == "random":
        p = g.uniform(-60, 60, (n, 3))
    elif case == "duplicates":                          # heavy duplication: ~4000 voxels for 300 000 rows
        p = g.uniform(-0.8, 0.8, (n, 3)) + g.integers(-4, 4, (n, 1)) * 10.0
    elif case == "negative":
        p = -g.uniform(0, 0.35, (n, 3))
    else:
        p = g.uniform(-60, 60, (n, 3))
        for v in (np.nan, np.inf, -np.inf):
            p[g.choice(n, n // 20, replace=False), g.integers(0, 3, n // 20)] = v
    got, status = voxel_first(p)
    ref, rstatus = F.restate_voxel_first(p, 0.1, 50.0)
    assert status == rstatus == 0 and got.shape == ref.shape
    np.testing.assert_array_equal(got, ref)


def test_voxel_first_flags_keys_out_of_range():
    p = np.array([[1.0, 2.0, 3.0], [2e5, 0.0, 0.0], [np.inf, 0.0, 0.0]])
    got, status = voxel_first(p)
    assert status == 1 and got.shape == (1, 3)
    assert voxel_first(np.zeros((0, 3)))[0].shape == (0, 3)


# ---- whole samples -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def data_root(tmp_path_factory):
    return G.make_dataset(str(tmp_path_factory.mktemp("kitti")))


@pytest.mark.parametrize("split", ["train", "validation", "test"])
def test_samples_match_the_reference(data_root, split):
    ds = R.TemporalKITTISet(data_root, G.SCAN_WINDOW, G.split_seqs(split), G.split_name(split), G.RESOLUTION, G.NUM_POINTS, "refine",
                            device=DEV)
    np.random.seed(G.SEED)
    torch.manual_seed(G.SEED)
    for k, i in enumerate(G.RECORD[split]):
        item = ds[i]
        assert item[0].device.type == "cuda" and item[3].device.type == "cuda"
        assert_close_to_golden(split, k, item)


# ---- Chamfer distance ----------------------------------------------------------------------------------------------------
def test_chamfer_per_point_against_brute_force_with_ties():
    g = np.random.default_rng(3)
    y = np.round(g.uniform(-2, 2, (2, 400, 3)), 1).astype(np.float32)      # a 0.1 lattice: many exact ties
    x = np.concatenate([np.round(g.uniform(-2, 2, (2, 300, 3)) * 20) / 20, y[:, :50]], 1).astype(np.float32)
    xt, yt = torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)
    for b in range(2):
        d2 = metrics._nn_sq_dist(xt[b], yt[b]).cpu().numpy()
        full = ((x[b].astype(np.float64)[:, None] - y[b].astype(np.float64)[None]) ** 2).sum(-1)
        j = full.argmin(1)                                                   # lowest index on ties
        ref = ((x[b] - y[b][j]) ** 2).sum(-1)
        np.testing.assert_allclose(d2, ref, rtol=2 ** -22, atol=0)
        assert (d2[300:] == 0).all()
    loss, normals = metrics.chamfer_distance(xt, yt)
    assert normals is None and loss.dtype == torch.float32 and loss.device.type == "cuda"


@pytest.mark.parametrize("b", [1, 2])
def test_chamfer_at_full_size_against_ckdtree(b):
    from scipy.spatial import cKDTree
    g = np.random.default_rng(b)
    y = g.uniform(-50, 50, (b, 360_000, 3)).astype(np.float32)
    x = (np.repeat(y[:, :180_000], 6, 1) + g.normal(0, 0.05, (b, 1_080_000, 3))).astype(np.float32)
    xt, yt = torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)
    loss, _ = metrics.chamfer_distance(xt, yt)
    cx, cy = [], []
    for k in range(b):
        dx, _ = cKDTree(y[k].astype(np.float64)).query(x[k].astype(np.float64), k=1)
        dy, _ = cKDTree(x[k].astype(np.float64)).query(y[k].astype(np.float64), k=1)
        gx = metrics._nn_sq_dist(xt[k], yt[k]).double().cpu().numpy()
        gy = metrics._nn_sq_dist(yt[k], xt[k]).double().cpu().numpy()
        np.testing.assert_allclose(gx, dx ** 2, rtol=2 ** -20, atol=1e-12)
        np.testing.assert_allclose(gy, dy ** 2, rtol=2 ** -20, atol=1e-12)
        cx.append((dx ** 2).mean())
        cy.append((dy ** 2).mean())
    ref = np.mean(cx) + np.mean(cy)
    assert abs(loss.item() - ref) <= 1e-6 * ref, (loss.item(), ref)


# ---- the CLI -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loader,write", [("val", False), ("test", True)])
def test_cli_end_to_end(data_root, tmp_path, loader, write):
    from lidiff_b200.tools import test_refine as T
    cfg = {"data": {"data_dir": data_root, "resolution": 0.05, "split": "train", "train": G.TRAIN, "validation": G.VALIDATION,
                    "scan_window": G.SCAN_WINDOW, "num_points": G.NUM_POINTS},
           "train": {"batch_size": 2, "num_workers": 4, "mode": "refine", "up_factor": 6}}
    path = tmp_path / "config_refine.yaml"
    path.write_text(yaml.safe_dump(cfg))
    args = ["--random-weights", "-c", str(path), "--loader", loader] + (["--out", str(tmp_path / "out")] if write else [])
    res = CliRunner().invoke(T.main, args, catch_exceptions=False)
    assert res.exit_code == 0, res.output
    tag = "test" if loader == "test" else "val"
    printed = [float(line.split()[-1]) for line in res.output.splitlines() if line.startswith("batch ")]
    # the same batches again, their loss computed directly through the ME surface and chamfer_distance
    from lidiff_b200.tools.test_completion import set_deterministic
    set_deterministic()
    net = T.load_refine_net(None, 6, torch.device(DEV), random_weights=True)
    dm = R.TemporalKittiDataModule(cfg, device=DEV)
    data = dm.test_dataloader() if loader == "test" else dm.val_dataloader()
    direct = []
    for batch in data:
        import lidiff_b200.me as ME
        with torch.no_grad():
            xf = ME.utils.batched_coordinates(list(batch["pcd_noise"]), dtype=torch.float32, device=DEV)
            x_t = ME.TensorField(features=xf[:, 1:], coordinates=torch.round(xf / 0.05), device=DEV)
            refined = (xf[:, None, 1:] + net(x_t).reshape(-1, 6, 3)).reshape(batch["pcd_full"].shape[0], -1, 3)
            direct.append(metrics.chamfer_distance(refined, batch["pcd_full"].to(DEV))[0].item())
    assert len(printed) == len(direct) == (5 if loader == "test" else 1)
    np.testing.assert_array_equal(np.float32(printed), np.float32(direct))
    assert f"{tag}/cd_loss mean over {len(direct)} batches" in res.output
    if write:
        plys = sorted(os.listdir(tmp_path / "out" / "refined" / "00"))
        assert plys == ["000000.ply", "000001.ply", "000002.ply", "000003.ply"]
        assert os.listdir(tmp_path / "out" / "refined" / "01") == ["000000.ply"]
