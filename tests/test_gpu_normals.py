"""Point normals on the GPU (lb2_pc_knn / lb2_pc_normals through lidiff_b200.normals) against the numpy restatement of open3d's
estimate_normals (tests/normals_oracle.py): exact k-NN rows and bit-exact squared distances, normals within 1e-9 of the restatement
wherever the eigenvector is well defined, exact signs wherever the solver's sign decisions have a margin, exact degenerate cases,
determinism, the open3d shim and the completion CLI's `--normals` output."""
import os

import numpy as np
import pytest
import torch

import normals_oracle as O
from lidiff_b200 import normals as N

pytestmark = pytest.mark.gpu


def _clouds():
    g = np.random.default_rng(7)
    return {"cube": g.uniform(-10, 10, (20_000, 3)),
            "slab": g.uniform(-10, 10, (20_000, 3)) * [1.0, 1.0, 0.001],
            "dup40": np.repeat(g.uniform(-5, 5, (500, 3)), 40, 0)[g.permutation(20_000)],
            "n_lt_k": g.uniform(-1, 1, (20, 3)),
            "n1": np.array([[0.25, -3.5, 7.0]])}


def _check_knn(p, k):
    idx, d2 = N.knn(p, k)
    want_i, want_d = O.knn(p, k)
    idx, d2 = idx.cpu().numpy(), d2.cpu().numpy()
    assert idx.shape == want_i.shape == (p.shape[0], min(k, p.shape[0]))
    assert np.array_equal(idx, want_i), f"{(idx != want_i).any(1).sum()} rows differ"
    assert np.array_equal(d2.view(np.int64), want_d.view(np.int64))        # bit for bit
    return idx


@pytest.mark.parametrize("k", [1, 8, 30, 32])
@pytest.mark.parametrize("cloud", ["cube", "slab", "dup40", "n_lt_k", "n1"])
def test_knn_rows_equal_the_restatement(cloud, k):
    p = _clouds()[cloud]
    idx = _check_knn(p, k)
    if cloud == "dup40":                                                # ties everywhere: the lowest indices of the copies win
        first = {}
        for i in range(p.shape[0]):
            first.setdefault(tuple(p[i]), []).append(i)
        for i in range(0, p.shape[0], 997):
            assert np.array_equal(idx[i], first[tuple(p[i])][:k])


def _check_normals(p, nrm, min_clear=None):
    want, diag, cov = O.normals_from_idx(p, O.knn(p, 30)[0])
    gap = O.eigen_gap(cov) >= 1e-6
    dots = (nrm * want).sum(1)
    assert (1 - np.abs(dots[gap])).max(initial=0.0) <= 1e-9
    clear = O.clear_sign(diag) & gap
    assert (dots[clear] > 0).all(), f"{(dots[clear] <= 0).sum()} clear points with the other sign"
    if min_clear is not None:
        assert clear.mean() >= min_clear, clear.mean()
    return want


def test_refined_like_cloud_knn_and_normals():
    p = O.refined_like()
    _check_knn(p, 30)
    nrm = N.estimate_normals(p).cpu().numpy()
    _check_normals(p, nrm, min_clear=0.99)


@pytest.mark.parametrize("cloud", ["cube", "slab"])
def test_normals_small_clouds(cloud):
    p = _clouds()[cloud]
    _check_normals(p, N.estimate_normals(p).cpu().numpy())


def test_degenerate_cases_match_exactly():
    g = np.random.default_rng(8)
    line = np.c_[g.uniform(-5, 5, 300), np.zeros(300), np.zeros(300)]                 # axis-aligned: no off-diagonal term
    dup = np.repeat(np.array([[1.5, -2.25, 0.75], [100.5, 3.0, -7.125]]), 40, 0)     # dyadic: exactly zero covariance
    for p in (line, dup, np.array([[0.0, 0.0, 0.0], [1.0, 2.0, 3.0]]), np.array([[1.0, 1.0, 1.0]])):
        want = O.estimate_normals(p)[0]
        assert np.array_equal(N.estimate_normals(p).cpu().numpy(), want)
    assert np.array_equal(N.estimate_normals(dup).cpu().numpy(), np.tile([0.0, 0.0, 1.0], (80, 1)))
    # a z = 0 plane: the trigonometric branch; x and y exactly zero, the restatement's sign on every point
    plane = np.c_[g.uniform(-1, 1, (3000, 2)), np.zeros(3000)]
    got, want = N.estimate_normals(plane).cpu().numpy(), O.estimate_normals(plane)[0]
    assert (got[:, :2] == 0).all() and np.array_equal(np.sign(got[:, 2]), np.sign(want[:, 2]))
    assert np.abs(got[:, 2] - want[:, 2]).max() <= 1e-15


def test_two_runs_give_identical_bits():
    p = torch.as_tensor(O.refined_like(1, 60_000), device="cuda")
    a, b = N.knn(p, 30), N.knn(p, 30)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int64), b[1].view(torch.int64))
    na, nb = N.estimate_normals(p), N.estimate_normals(p)
    assert torch.equal(na.view(torch.int64), nb.view(torch.int64))


def test_k_over_32_is_unsupported_by_the_library():
    from lidiff_b200 import _lib
    h = _lib.get_handle("cuda")
    p = torch.as_tensor(_clouds()["cube"][:100], device="cuda")
    idx = torch.empty((100, 33), dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="-3"):
        h.pc_knn(h.pc_tree(p), 100, 33, idx)
    with pytest.raises(ValueError):
        N.estimate_normals(p, knn=33)


def test_non_finite_points_leave_empty_slots_and_nan_normals():
    """a NaN or infinite point gets an empty neighbour row (-1, +inf) and a NaN normal, nothing reads outside the cloud, and the
    finite points keep exactly the neighbours and normals they have without those points"""
    g = np.random.default_rng(9)
    fin = g.uniform(-3, 3, (3000, 3))
    bad = np.array([[np.nan, 0.0, 0.0], [0.0, np.inf, 0.0], [-np.inf, 1.0, 2.0], [1.0, 2.0, -np.nan]])
    pos = np.sort(g.choice(3000 + 4, 4, replace=False))
    p = np.empty((3004, 3))
    is_bad = np.zeros(3004, bool)
    is_bad[pos] = True
    p[is_bad], p[~is_bad] = bad, fin
    keep = np.flatnonzero(~is_bad)                                      # finite-cloud index -> mixed-cloud index
    for k in (8, 30):
        idx, d2 = (t.cpu().numpy() for t in N.knn(p, k))
        assert (idx[is_bad] == -1).all() and np.isinf(d2[is_bad]).all()
        want_i, want_d = O.knn(fin, k)
        assert np.array_equal(idx[~is_bad], keep[want_i]) and np.array_equal(d2[~is_bad], want_d)
    nrm = N.estimate_normals(p).cpu().numpy()
    assert np.isnan(nrm[is_bad]).all()
    assert np.array_equal(nrm[~is_bad], N.estimate_normals(fin).cpu().numpy())
    # fewer finite points than k: the finite points' rows end in empty slots too, and their normals are NaN
    few = np.concatenate([g.uniform(-1, 1, (5, 3)), np.full((3, 3), np.nan)])
    idx, d2 = (t.cpu().numpy() for t in N.knn(few, 8))
    assert (idx[:5, :5] >= 0).all() and (idx[:5, 5:] == -1).all() and np.isinf(d2[:5, 5:]).all() and (idx[5:] == -1).all()
    assert np.isnan(N.estimate_normals(few, knn=8).cpu().numpy()).all()
    torch.cuda.synchronize()


def test_knn_with_another_clouds_point_count_writes_empty_rows():
    from lidiff_b200 import _lib
    h = _lib.get_handle("cuda")
    p = torch.as_tensor(_clouds()["cube"][:100], device="cuda")
    tree = h.pc_tree(p)
    for n in (60, 140):
        idx = torch.zeros((n, 8), dtype=torch.int32, device="cuda")
        d2 = torch.zeros((n, 8), dtype=torch.float64, device="cuda")
        h.pc_knn(tree, n, 8, idx, d2)
        assert (idx == -1).all() and torch.isinf(d2).all()


def test_shim_replays_the_reference_scripts_output_step(tmp_path):
    """the reference's inference script ends every scan with (tools/diff_completion_pipeline.py:204-212)
        pcd = o3d.geometry.PointCloud(); pcd.points = o3d.utility.Vector3dVector(scan); pcd.estimate_normals()
        o3d.io.write_point_cloud(path, pcd)
    for the refined and the diffusion cloud.  The reference's script itself is not part of this repository and cannot be imported
    where the GPU tests run (tests/test_reference_on_shims.py works from a recorded golden for the same reason), so this test runs
    those lines through the shim on the two clouds the mirror (lidiff_b200.pipeline.DiffCompletion, which reproduces the reference
    class bit for bit) computes for a small scan at T = 2.  The PLYs they write carry normals equal bit for bit to
    lidiff_b200.normals.estimate_normals of their points."""
    from lidiff_b200 import shims
    from lidiff_b200.pipeline import DiffCompletion
    from lidiff_b200.synth import range_filter, synthetic_scan
    from test_reference_on_shims import lightning_checkpoints
    shims.install()
    import open3d as o3d
    diff_path, refine_path = lightning_checkpoints(tmp_path, 2000)
    pipe = DiffCompletion(diff_path, refine_path, 2, 6.0, device="cuda")
    refine_scan, diff_scan = pipe.complete_scan(range_filter(synthetic_scan(9, beams=16, azimuths=256)))
    for name, scan in (("refine", refine_scan), ("diff", diff_scan)):
        pcd = o3d.geometry.PointCloud()
        pcd.points = o3d.utility.Vector3dVector(scan)
        pcd.estimate_normals()
        path = str(tmp_path / f"{name}.ply")
        o3d.io.write_point_cloud(path, pcd)
        back = o3d.io.read_point_cloud(path)
        assert back.has_normals() and np.array_equal(np.asarray(back.points), scan)
        want = N.estimate_normals(np.asarray(back.points)).cpu().numpy()
        assert np.array_equal(np.asarray(back.normals).view(np.int64), want.view(np.int64))


def test_cli_writes_normals_matching_the_restatement(tmp_path):
    from click.testing import CliRunner
    from lidiff_b200.synth import synthetic_scan
    from lidiff_b200.tools import diff_completion_pipeline as P
    import lidiff_b200.shims.open3d as o3d
    scans = tmp_path / "scans"
    scans.mkdir()
    np.c_[synthetic_scan(3, beams=32, azimuths=1024), np.ones(32 * 1024)].astype(np.float32).tofile(scans / "000000.bin")
    out = tmp_path / "out"
    res = CliRunner().invoke(P.main, ["--path", str(scans), "--out", str(out), "--random-weights", "--normals", "-T", "2"],
                             catch_exceptions=False)
    assert res.exit_code == 0, res.output
    for kind in ("refine", "diff"):
        (f,) = [os.path.join(r, x) for r, _, fs in os.walk(out) for x in fs if r.endswith(kind) and x.endswith(".ply")]
        back = o3d.io.read_point_cloud(f)
        assert back.has_normals() and len(back.points) > 1000
        _check_normals(np.asarray(back.points), np.asarray(back.normals))
