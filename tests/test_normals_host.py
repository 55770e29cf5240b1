"""Point normals without a GPU: known answers of the numpy restatement of open3d's estimate_normals (tests/normals_oracle.py), and
the host logic of lidiff_b200.normals, the open3d shim's PLY round trip, the completion CLI's `--normals` output and eval_path's
file mode on the CPU stand-ins of tests/fake_normals_backend.py."""
import os
import shutil

import numpy as np
import pytest
import torch
from click.testing import CliRunner

import fake_normals_backend
import normals_oracle as O
from lidiff_b200 import normals as N
from lidiff_b200.synth import read_ply_xyz


@pytest.fixture
def fake(monkeypatch):
    return fake_normals_backend.install(monkeypatch)


# ---- the restatement ------------------------------------------------------------------------------------------------------------
def test_plane_gives_the_solvers_sign_of_z():
    g = np.random.default_rng(0)
    p = np.c_[g.uniform(-1, 1, (400, 2)), np.zeros(400)]
    nrm, diag, cov, idx, _ = O.estimate_normals(p)
    assert (cov[:, 2, :] == 0).all() and (cov[:, :, 2] == 0).all()
    assert np.array_equal(np.abs(nrm[:, :2]), np.zeros((400, 2))) and np.abs(np.abs(nrm[:, 2]) - 1).max() <= 1e-15
    # FastEigen3x3 on a z = 0 plane with in-plane eigenvalues l1 <= l2: half_det >= 0 exactly when l2 >= 2 l1.  Then the normal is
    # evec1 x evec2 = -U, where U = +-z is picked by ComputeEigenvector1 from the sign of evec2's larger component, which is always
    # the one that makes the result -z.  Otherwise ComputeEigenvector0's winning cross product is row0 x row1 = (0, 0, det) with
    # det > 0: +z.
    w = np.linalg.eigvalsh(cov[:, :2, :2])
    clear = np.abs(w[:, 1] / w[:, 0] - 2) > 1e-6
    assert clear.mean() > 0.95 and (diag["half_det"][clear] > 0).all()
    assert np.array_equal(np.sign(nrm[clear, 2]), np.where(w[clear, 1] > 2 * w[clear, 0], -1.0, 1.0))
    nrm, _ = O.fast_eigen3x3(np.array([[[4.0, 0.5, 0], [0.5, 1, 0], [0, 0, 0]], [[1.0, 0.5, 0], [0.5, 4, 0], [0, 0, 0]],
                                       [[4.0, -0.5, 0], [-0.5, 1, 0], [0, 0, 0]], [[1.0, 0.1, 0], [0.1, 1.2, 0], [0, 0, 0]]]))
    assert np.array_equal(nrm, [[0, 0, -1], [0, 0, -1], [0, 0, -1], [0, 0, 1]])


def test_axis_aligned_covariances_give_the_smallest_axis():
    covs = np.array([np.diag([3.0, 1.0, 2.0]), np.diag([1.0, 2.0, 3.0]), np.diag([2.0, 3.0, 0.5]), np.diag([1.0, 1.0, 2.0])])
    nrm, diag = O.fast_eigen3x3(covs)
    assert np.array_equal(nrm, [[0, 1, 0], [1, 0, 0], [0, 0, 1], [0, 0, 1]])   # a tie between x and y: neither is strictly smallest
    assert (diag["half_det"] == 0).all()                                         # the off-diagonal branch, no trigonometry


def test_fewer_than_three_neighbours_give_the_identity_and_z():
    p = np.array([[0.0, 0.0, 0.0], [1.0, 2.0, 3.0]])
    nrm, _, cov, idx, _ = O.estimate_normals(p)
    assert idx.shape == (2, 2) and (cov == np.eye(3)).all()
    assert np.array_equal(nrm, [[0, 0, 1], [0, 0, 1]])
    nrm, _, cov = O.normals_from_idx(np.random.default_rng(0).normal(size=(10, 3)), np.tile(np.arange(2), (10, 1)))
    assert (cov == np.eye(3)).all() and (nrm == [0, 0, 1]).all()


def test_all_duplicate_neighbourhood_gives_zero_covariance_and_z():
    # dyadic coordinates: the cumulants are exact, so E[pp^T] - E[p]E[p]^T is exactly 0 and the solver returns the zero vector
    base = np.array([[1.5, -2.25, 0.75], [100.5, 3.0, -7.125]])
    p = np.repeat(base, 40, 0)
    nrm, _, cov, idx, d2 = O.estimate_normals(p)
    assert (cov == 0).all() and (nrm == [0, 0, 1]).all()
    assert np.array_equal(idx[0], np.arange(30)) and np.array_equal(idx[45], 40 + np.arange(30)) and (d2 == 0).all()


def test_random_spd_matrices_agree_with_eigh_up_to_sign():
    g = np.random.default_rng(1)
    m = g.normal(size=(5000, 3, 3)) * g.uniform(1e-3, 1e3, (5000, 1, 1))
    cov = m @ m.transpose(0, 2, 1)
    nrm, _ = O.fast_eigen3x3(cov)
    w, v = np.linalg.eigh(cov)
    ok = (w[:, 1] - w[:, 0]) / w[:, 2] >= 1e-6
    assert ok.mean() > 0.99
    assert np.abs(np.linalg.norm(nrm, axis=1) - 1).max() <= 1e-12
    assert (1 - np.abs((nrm[ok] * v[ok, :, 0]).sum(1))).max() <= 1e-9


def test_restated_knn_orders_by_distance_then_index():
    g = np.random.default_rng(2)
    ax = np.arange(4, dtype=np.float64)
    lat = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)[g.permutation(64)]      # many exact ties
    idx, d2 = O.knn(lat, 10)
    full = ((lat[:, None, :] - lat[None]) ** 2).sum(-1)
    want = np.lexsort((np.broadcast_to(np.arange(64), (64, 64)), full), axis=1)[:, :10]
    assert np.array_equal(idx, want) and np.array_equal(d2, np.take_along_axis(full, want, 1))


# ---- lidiff_b200.normals on the CPU stand-ins -----------------------------------------------------------------------------------
def test_knn_and_normals_shapes_dtypes_and_errors(fake):
    g = np.random.default_rng(3)
    p = g.normal(size=(200, 3))
    idx, d2 = N.knn(p, 8)
    assert idx.shape == (200, 8) and idx.dtype == torch.int32 and d2.shape == (200, 8) and d2.dtype == torch.float64
    want_i, want_d = O.knn(p, 8)
    assert np.array_equal(idx.numpy(), want_i) and np.array_equal(d2.numpy(), want_d)
    nrm = N.estimate_normals(torch.from_numpy(p).float())                     # fp32 torch input: promoted to fp64
    assert nrm.shape == (200, 3) and nrm.dtype == torch.float64
    assert np.array_equal(nrm.numpy(), O.estimate_normals(p.astype(np.float32).astype(np.float64))[0])
    idx, _ = N.knn(p[:5], 30)                                                  # n < k: k_eff = n
    assert idx.shape == (5, 5)
    for k in (0, 33):
        with pytest.raises(ValueError):
            N.knn(p, k)
        with pytest.raises(ValueError):
            N.estimate_normals(p, knn=k)
    with pytest.raises(ValueError):
        N.estimate_normals(np.zeros((4, 2)))
    idx, d2 = N.knn(np.zeros((0, 3)), 30)
    assert idx.shape == (0, 0) and d2.shape == (0, 0)
    assert N.estimate_normals(np.zeros((0, 3))).shape == (0, 3)


def test_shim_point_cloud_is_accepted(fake):
    import lidiff_b200.shims.open3d as o3d
    p = np.random.default_rng(4).normal(size=(50, 3))
    assert np.array_equal(N.estimate_normals(o3d.geometry.PointCloud(p)).numpy(), O.estimate_normals(p)[0])


# ---- PLY files: the CLI writer, the shim reader, eval_path's reader -------------------------------------------------------------
def _old_writer_bytes(pts):
    pts = np.ascontiguousarray(pts, dtype=np.float64)
    return (("ply\nformat binary_little_endian 1.0\ncomment Created by lidiff_b200\n"
             f"element vertex {pts.shape[0]}\nproperty double x\nproperty double y\nproperty double z\nend_header\n").encode("ascii")
            + pts.astype("<f8").tobytes())


def test_ply_with_normals_round_trips_through_the_shim_and_read_ply_xyz(tmp_path):
    import lidiff_b200.shims.open3d as o3d
    from lidiff_b200.tools.diff_completion_pipeline import write_ply
    g = np.random.default_rng(5)
    p, n = g.normal(size=(123, 3)), g.normal(size=(123, 3))
    write_ply(str(tmp_path / "a.ply"), p)
    assert (tmp_path / "a.ply").read_bytes() == _old_writer_bytes(p)
    write_ply(str(tmp_path / "b.ply"), p, n)
    back = o3d.io.read_point_cloud(str(tmp_path / "b.ply"))
    assert back.has_normals() and np.array_equal(np.asarray(back.points), p) and np.array_equal(np.asarray(back.normals), n)
    assert np.array_equal(read_ply_xyz(str(tmp_path / "b.ply")), p)
    # the shim's own writer gives the same vertex bytes
    pc = o3d.geometry.PointCloud(p)
    pc.normals = n
    o3d.io.write_point_cloud(str(tmp_path / "c.ply"), pc)
    body = lambda f: (tmp_path / f).read_bytes().split(b"end_header\n", 1)[1]
    assert body("b.ply") == body("c.ply")
    with pytest.raises(ValueError):
        write_ply(str(tmp_path / "d.ply"), p, n[:5])


class _StubCompletion:
    """stands in for lidiff_b200.pipeline.DiffCompletion: a fixed (refined, diffusion) pair per scan"""

    def __init__(self, *a, **k):
        pass

    def complete_scan(self, points):
        g = np.random.default_rng(points.shape[0])
        post = points[: points.shape[0] // 2] + g.normal(0, 0.01, (points.shape[0] // 2, 3))
        return (post[:, None, :] + g.normal(0, 0.03, (post.shape[0], 6, 3))).reshape(-1, 3), post


def _run_cli(monkeypatch, tmp_path, scans, extra):
    from lidiff_b200.tools import diff_completion_pipeline as P
    monkeypatch.setattr(P, "DiffCompletion", _StubCompletion)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    out = tmp_path / "out"
    res = CliRunner().invoke(P.main, ["--path", str(scans), "--out", str(out), "-T", "2"] + extra, catch_exceptions=False)
    assert res.exit_code == 0, res.output
    return out / "diff_net_T2_s6.0"


def test_cli_normals_flag(fake, monkeypatch, tmp_path):
    from lidiff_b200.synth import synthetic_scan
    scans = tmp_path / "scans"
    scans.mkdir()
    for b in range(2):
        np.c_[synthetic_scan(b, beams=8, azimuths=64), np.ones(512)].astype(np.float32).tofile(scans / f"{b:06d}.bin")
    plain = _run_cli(monkeypatch, tmp_path / "a", scans, [])
    with_n = _run_cli(monkeypatch, tmp_path / "b", scans, ["--normals"])
    import lidiff_b200.shims.open3d as o3d
    for b in range(2):
        pts = np.fromfile(scans / f"{b:06d}.bin", dtype=np.float32).reshape(-1, 4)[:, :3]
        refined, post = _StubCompletion().complete_scan(pts)
        for kind, cloud in (("refine", refined), ("diff", post)):
            assert (plain / kind / f"{b:06d}.ply").read_bytes() == _old_writer_bytes(cloud)      # no flag: today's bytes
            back = o3d.io.read_point_cloud(str(with_n / kind / f"{b:06d}.ply"))
            assert np.array_equal(np.asarray(back.points), cloud)
            assert np.array_equal(np.asarray(back.normals), O.estimate_normals(cloud)[0])


def test_eval_path_scores_files_with_and_without_normals_alike(monkeypatch, tmp_path):
    import fake_metrics_backend
    from eval_sequence import make_sequence
    from lidiff_b200.tools import eval_path as E
    from lidiff_b200.tools.diff_completion_pipeline import write_ply
    fake_metrics_backend.install(monkeypatch)
    seq, pred = make_sequence(str(tmp_path))
    pred_n = str(tmp_path / "pred_normals")
    shutil.copytree(pred, pred_n)
    g = np.random.default_rng(6)
    for f in os.listdir(pred_n):
        p = read_ply_xyz(os.path.join(pred_n, f))
        write_ply(os.path.join(pred_n, f), p, g.normal(size=p.shape))
    _, a = E.score_scans(seq, pred, None, 50.0, "refine", "cpu")
    _, b = E.score_scans(seq, pred_n, None, 50.0, "refine", "cpu")
    assert sorted(a) == sorted(b) == [0, 1, 2]
    assert all(torch.equal(a[k], b[k]) for k in a)
