"""Host tests of mesh sampling: the restatement of open3d's SamplePointsUniformly (tests/mesh_reference.py) pinned by hand-checked
cases and by a literal transcription of open3d's loop, the MT19937 seeding, the host logic of lidiff_b200.mesh, the open3d shim's
TriangleMesh, utility.random and read_triangle_mesh, Metrics3D and `eval_path --mesh`, on the CPU stand-in backend
(tests/fake_mesh_backend.py)."""
import json
import os

import numpy as np
import pytest
import torch

import fake_mesh_backend
import mesh_reference as MR
import rng_reference as R
from eval_sequence import make_sequence
from lidiff_b200 import mesh as MESH
from lidiff_b200 import metrics as M
from lidiff_b200.shims.open3d import geometry, io, utility
from lidiff_b200.tools import eval_path as E
from lidiff_b200.tools.diff_completion_pipeline import write_ply
from mesh_files import mesh_prediction, write_mesh_ply, write_mesh_predictions

UNIT = (np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), np.array([[0, 1, 2]], np.int32))


@pytest.fixture
def fake(monkeypatch):
    return fake_mesh_backend.install(monkeypatch)


def _words(seed, n):
    return R.mt_words(*MESH.seed_state(seed), n)[0]


# ---- the restatement ----------------------------------------------------------------------------------------------------------
def test_mt19937_check_values():
    mt = np.random.MT19937()
    mt._legacy_seeding(5489)
    assert mt.random_raw(10000)[-1] == 4123659995                  # the C++ standard's check value of std::mt19937
    key, pos = MESH.seed_state(5489)
    assert pos == 624 and R.mt_words(key, pos, 10000)[0][-1] == 4123659995
    assert np.array_equal(MESH.seed_state(-1)[0], MESH.seed_state(2 ** 32 - 1)[0])     # libstdc++ takes the seed modulo 2^32


def test_canonical_and_its_guard():
    assert MR.canonical(0, 0) == 0.0
    assert MR.canonical(1, 0) == 2.0 ** -64
    assert MR.canonical(0, 1) == 2.0 ** -32
    assert MR.canonical(0xFFFFFFFF, 0xFFFFFFFF) == np.nextafter(1.0, 0.0)          # RN(2^64 - 1) = 2^64: the guard
    assert MR.canonical(0xFFFFF800, 0xFFFFFFFF) < 1.0


def test_round_half_away_from_zero():
    x = np.array([0.0, 0.5, 1.5, 2.5, 0.49999999999999994, 3.4999999999999996, 1e15 + 0.5])
    assert MR.round_half_away(x).tolist() == [0.0, 1.0, 2.0, 3.0, 0.0, 3.0, 1e15 + 1.0]


def test_one_triangle_every_point_inside():
    v, t = UNIT
    n = 2000
    w = _words(1, 4 * n)
    p = MR.sample(v, t, n, w)
    assert (p[:, 2] == 0).all() and (p[:, :2] >= 0).all() and (p[:, 0] + p[:, 1] <= 1.0 + 1e-15).all()
    r1, r2 = MR.canonical(w[0::4], w[1::4]), MR.canonical(w[2::4], w[3::4])
    s = np.sqrt(r1)
    assert np.abs((1.0 - s) + s * (1.0 - r2) + s * r2 - 1.0).max() <= 4e-16
    assert np.array_equal(p[:, 0], s * (1.0 - r2)) and np.array_equal(p[:, 1], s * r2)      # v1 = e_x, v2 = e_y


def test_areas_one_to_three_and_four_points():
    v = np.array([[0.0, 0, 0], [1, 0, 0], [0, 2, 0], [5, 0, 0], [8, 0, 0], [5, 2, 0]])
    t = np.array([[0, 1, 2], [3, 4, 5]])
    a = MR.areas(v, t)
    assert a.tolist() == [1.0, 3.0] and MR.surface_area(a) == 4.0
    n_t = MR.counts(a, 4)
    assert n_t.tolist() == [1, 4] and np.diff(np.concatenate([[0], n_t])).tolist() == [1, 3]
    p = MR.sample(v, t, 4, _words(2, 16))
    assert (p[0, 0] <= 1.0) and (p[1:, 0] >= 5.0).all()


def test_zero_area_triangles_get_no_points():
    v = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 2, 2]])
    t = np.array([[0, 0, 1], [0, 1, 2], [3, 3, 3], [0, 1, 1], [1, 2, 0], [0, 3, 3]])
    a = MR.areas(v, t)
    assert a.tolist() == [0.0, 0.5, 0.0, 0.0, 0.5, 0.0]
    n_t = MR.counts(a, 1001)
    owned = np.diff(np.concatenate([[0], n_t]))
    assert owned[[0, 2, 3, 5]].tolist() == [0, 0, 0, 0] and owned.sum() == 1001
    assert owned.tolist() == [0, 501, 0, 0, 500, 0]                   # round(0.5 * 1001) = 501, half away from zero


def test_fewer_points_than_triangles():
    v, t = MR.height_field(6, seed=3)                                # 50 triangles
    for n in (1, 3, 7):
        n_t = MR.counts(MR.areas(v, t), n)
        assert n_t[-1] == n and (np.diff(n_t) >= 0).all()
        assert np.array_equal(MR.sample(v, t, n, _words(n, 4 * n)), MR.sample_loop(v, t, n, _words(n, 4 * n)))


def test_all_ones_words_take_the_guard():
    v = np.array([[1.0, 2.0, 3.0], [4.0, -1.0, 0.5], [-2.0, 0.25, 7.0]])
    t = np.array([[0, 1, 2]])
    n = 5
    w = np.full(4 * n, 0xFFFFFFFF, np.uint32)
    p = MR.sample(v, t, n, w)
    assert np.array_equal(p, MR.sample_loop(v, t, n, w))
    s = np.sqrt(np.nextafter(1.0, 0.0))
    a, b, c = 1.0 - s, s * (1.0 - np.nextafter(1.0, 0.0)), s * np.nextafter(1.0, 0.0)
    assert np.array_equal(p[0], (a * v[0] + b * v[1]) + c * v[2])
    assert np.isfinite(p).all()


@pytest.mark.parametrize("seed", range(4))
def test_vectorised_restatement_equals_open3ds_loop(seed):
    g = np.random.default_rng(seed)
    v = g.normal(0, 10, (40, 3)) + (1e5 if seed % 2 else 0.0)
    t = g.integers(0, 40, (60, 3))
    t[::7, 1] = t[::7, 0]                                           # degenerate triangles
    n = int(g.integers(1, 500))
    w = _words(seed, 4 * n)
    assert np.array_equal(MR.sample(v, t, n, w), MR.sample_loop(v, t, n, w))


def test_sequential_sums_are_left_to_right():
    a = np.array([1e16, 1.0, 1.0, 3.0, 0.5])
    s = 0.0
    for x in a:
        s += x
    assert MR.surface_area(a) == s == (((1e16 + 1.0) + 1.0) + 3.0) + 0.5 != float(np.sum(a[::-1]))


# ---- lidiff_b200.mesh on the CPU stand-in -------------------------------------------------------------------------------------
def test_sample_points_uniformly_returns_the_restated_points_and_state(fake):
    v, t = MR.height_field(12, seed=1)
    key, pos = MESH.seed_state(9)
    pts, key2, pos2 = MESH.sample_points_uniformly(v, t, 333, key, pos, device="cpu")
    want, wkey, wpos = MR.sample_stream(v, t, 333, key, pos)
    assert np.array_equal(pts.numpy(), want) and np.array_equal(key2, wkey) and pos2 == wpos
    # the next call continues the stream
    pts2, _, _ = MESH.sample_points_uniformly(v, t, 50, key2, pos2, device="cpu")
    assert np.array_equal(pts2.numpy(), MR.sample_stream(v, t, 50, wkey, wpos)[0])


def _bad_meshes():
    v, t = UNIT
    nan = v.copy()
    nan[1, 2] = np.nan
    return [
        ("number_of_points", v, t, 0, ValueError),
        ("number_of_points", v, t, -3, ValueError),
        ("no triangles", v, np.zeros((0, 3), np.int32), 10, ValueError),
        ("outside", v, np.array([[0, 1, 3]], np.int32), 10, ValueError),
        ("outside", v, np.array([[0, -1, 2]], np.int32), 10, ValueError),
        ("outside", v, np.array([[0, 1, 2 ** 40]], np.int64), 10, ValueError),
        ("NaN or infinite", nan, t, 10, ValueError),
        ("surface area", v, np.array([[0, 0, 1], [2, 2, 2]], np.int32), 10, ValueError),
        ("surface area", np.array([[0.0, 0, 0], [1e300, 0, 0], [0, 1e300, 0]]), t, 10, ValueError),   # S = inf
    ]


@pytest.mark.parametrize("case", range(9))
def test_bad_input_raises_before_any_sampling(fake, case):
    what, v, t, n, exc = _bad_meshes()[case]
    key, pos = MESH.seed_state(4)
    launches = fake.launches
    with pytest.raises(exc, match=what):
        MESH.sample_points_uniformly(v, t, n, key, pos, device="cpu")
    assert fake.launches - launches <= 5                            # at most the prepare call, never the sampling kernel
    MESH.STREAM.seed(4)
    with pytest.raises(exc):
        MESH.STREAM.sample_points_uniformly(v, t, n, device="cpu")
    k2, p2 = MESH.STREAM.state()
    assert np.array_equal(k2, key) and p2 == pos                      # the stream did not move


def test_bad_count_status_raises_runtime_error(fake, monkeypatch):
    real = fake.mesh_sample_prepare

    def short(verts, tris, n_points, area, info, scratch):
        real(verts, tris, n_points, area, info, scratch)
        rec = np.frombuffer(info.numpy().tobytes(), fake_mesh_backend._INFO).copy()
        rec["status"] |= 8
        rec["last_count"] = n_points - 1
        info[:] = torch.from_numpy(rec.view(np.uint8))
    monkeypatch.setattr(fake, "mesh_sample_prepare", short)
    with pytest.raises(RuntimeError, match="hold 9 of the 10 points"):
        MESH.sample_points_uniformly(*UNIT, 10, *MESH.seed_state(0), device="cpu")


# ---- the open3d shim -------------------------------------------------------------------------------------------------------------
def test_triangle_mesh_surface(fake):
    v, t = MR.height_field(5, seed=2)
    m = geometry.TriangleMesh()
    assert not m.has_triangles() and m.get_geometry_type().value == 6 == geometry.GeometryType.TriangleMesh.value
    m.vertices = utility.Vector3dVector(v)
    m.triangles = utility.Vector3iVector(t)
    assert m.has_triangles() and np.asarray(m.triangles).dtype == np.int32 and len(m.vertices) == 25
    assert m.get_surface_area() == MR.surface_area(MR.areas(v, t))
    with pytest.raises(NotImplementedError):
        m.sample_points_uniformly(10, use_triangle_normal=True)
    with pytest.raises(RuntimeError):
        utility.Vector3iVector(np.zeros((2, 3)))
    with pytest.raises(RuntimeError):
        utility.Vector3iVector(np.array([[0, 1, 2 ** 33]]))


def test_global_stream_advances_by_4n(fake):
    v, t = MR.height_field(8, seed=5)
    utility.random.seed(42)
    m = geometry.TriangleMesh(v, t)
    a = np.asarray(m.sample_points_uniformly(1000).points)
    b = np.asarray(m.sample_points_uniformly(number_of_points=77).points)
    key, pos = MESH.seed_state(42)
    words, key2, pos2 = R.mt_words(key, pos, 4 * 1077)
    assert np.array_equal(a, MR.sample(v, t, 1000, words[:4000])) and np.array_equal(b, MR.sample(v, t, 77, words[4000:]))
    k, p = MESH.STREAM.state()
    assert np.array_equal(k, key2) and p == pos2
    assert np.asarray(m.sample_points_uniformly().points).shape == (100, 3)          # open3d's default
    with pytest.raises(TypeError):
        utility.random.seed(2 ** 31)


def test_draw_geometries_refuses_meshes():
    from lidiff_b200.shims.open3d import visualization
    with pytest.raises(NotImplementedError):
        visualization.draw_geometries([geometry.TriangleMesh(*UNIT)])


# ---- read_triangle_mesh -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian"])
@pytest.mark.parametrize("count,index,name,vtype", [("uchar", "int", "vertex_indices", "double"), ("int", "uint", "vertex_index", "float"),
                                                     ("uint", "int", "vertex_indices", "float"), ("uchar", "uint", "vertex_index", "double")])
def test_read_triangle_mesh_layouts(tmp_path, fmt, count, index, name, vtype):
    v, t = mesh_prediction(0)
    path = write_mesh_ply(str(tmp_path / "m.ply"), v, t, fmt=fmt, vtype=vtype, count=count, index=index, name=name)
    m = io.read_triangle_mesh(path)
    want = v.astype(np.float32).astype(np.float64) if vtype == "float" else v
    assert np.array_equal(np.asarray(m.vertices), want) and np.array_equal(np.asarray(m.triangles), t)
    assert np.asarray(m.triangles).dtype == np.int32
    pcd = io.read_point_cloud(path)                                 # the point reader still returns the vertices
    assert np.array_equal(np.asarray(pcd.points), want)


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian"])
def test_read_triangle_mesh_rejections(tmp_path, fmt):
    v, t = UNIT
    v4 = np.concatenate([v, [[1.0, 1.0, 0.0]]])
    quad = write_mesh_ply(str(tmp_path / "q.ply"), v4, [[0, 1, 2], [1, 3, 2, 0], [0, 1, 2]], fmt=fmt)
    with pytest.raises(RuntimeError, match="face 1 has 4 vertices"):
        io.read_triangle_mesh(quad)
    ok = write_mesh_ply(str(tmp_path / "ok.ply"), v, t, fmt=fmt)
    with pytest.raises(NotImplementedError):
        io.read_triangle_mesh(ok, enable_post_processing=True)
    extra = write_mesh_ply(str(tmp_path / "e.ply"), v, t, fmt=fmt, extra_header="property uchar red\n")
    with pytest.raises(RuntimeError, match="one property"):
        io.read_triangle_mesh(extra)
    edge = write_mesh_ply(str(tmp_path / "edge.ply"), v, t, fmt=fmt, extra_header="element edge 0\nproperty int vertex1\n")
    with pytest.raises(RuntimeError, match="vertex element"):
        io.read_triangle_mesh(edge)
    with pytest.raises(RuntimeError, match="one property"):
        io.read_triangle_mesh(write_mesh_ply(str(tmp_path / "s.ply"), v, t, fmt=fmt, count="short"))
    with pytest.raises(RuntimeError, match="one property"):
        io.read_triangle_mesh(write_mesh_ply(str(tmp_path / "f.ply"), v, t, fmt=fmt, index="float"))
    data = open(ok, "rb").read()
    open(tmp_path / "short.ply", "wb").write(data[:-3])
    with pytest.raises(RuntimeError, match="ends before" if fmt != "ascii" else "face 0 is malformed"):
        io.read_triangle_mesh(str(tmp_path / "short.ply"))
    open(tmp_path / "not.ply", "wb").write(b"off\n")
    with pytest.raises(RuntimeError, match="not a PLY"):
        io.read_triangle_mesh(str(tmp_path / "not.ply"))


def test_read_triangle_mesh_of_a_point_cloud_file(tmp_path):
    write_ply(str(tmp_path / "p.ply"), np.arange(12.0).reshape(4, 3))
    m = io.read_triangle_mesh(str(tmp_path / "p.ply"))
    assert np.asarray(m.vertices).shape == (4, 3) and not m.has_triangles()


# ---- Metrics3D ---------------------------------------------------------------------------------------------------------------
def test_metrics3d_conversions(fake):
    m3 = M.Metrics3D()
    pts = np.random.default_rng(0).normal(size=(50, 4))
    pcd = geometry.PointCloud(pts[:, :3])
    assert m3.convert_to_pcd(pcd) is pcd and not m3.prediction_is_empty(pcd)
    assert m3.prediction_is_empty(geometry.PointCloud())
    for x in (pts, torch.from_numpy(pts)):
        out = m3.convert_to_pcd(x)
        assert isinstance(out, geometry.PointCloud) and np.array_equal(np.asarray(out.points), pts[:, :3])
        assert not m3.prediction_is_empty(x) and m3.prediction_is_empty(x[:0])
    v, t = MR.height_field(10, seed=8)
    mesh = geometry.TriangleMesh(v, t)
    assert not m3.prediction_is_empty(mesh)
    assert m3.prediction_is_empty(geometry.TriangleMesh(v, None)) and m3.prediction_is_empty(geometry.TriangleMesh(None, None))
    utility.random.seed(3)
    out = m3.convert_to_pcd(mesh)
    assert np.array_equal(np.asarray(out.points), MR.sample_stream(v, t, 1000000, *MESH.seed_state(3))[0])
    with pytest.raises(TypeError):
        m3.convert_to_pcd([1, 2, 3])
    with pytest.raises(TypeError):
        m3.prediction_is_empty(geometry.VoxelGrid())
    assert isinstance(M.PrecisionRecall(*M.PR_ARGS), M.Metrics3D)


def test_metrics3d_takes_the_shim_under_its_open3d_name(fake):
    import lidiff_b200.shims as sh
    sh.install()
    import open3d as o3d
    mesh = o3d.geometry.TriangleMesh(o3d.utility.Vector3dVector(UNIT[0]), o3d.utility.Vector3iVector(UNIT[1]))
    o3d.utility.random.seed(11)
    p = np.asarray(M.Metrics3D.convert_to_pcd(mesh).points)
    assert np.array_equal(p, MR.sample_stream(*UNIT, 1000000, *MESH.seed_state(11))[0])


# ---- eval_path --mesh ---------------------------------------------------------------------------------------------------------
def test_eval_path_mesh_equals_scoring_the_restated_samples(fake, tmp_path, monkeypatch):
    n = 20000                                                       # the CPU stand-in's size; the GPU test samples 10^6 points
    monkeypatch.setattr(M, "MESH_SAMPLES", n)
    seq, pred = make_sequence(str(tmp_path))
    write_mesh_predictions(pred)
    pts_dir = tmp_path / "points"
    pts_dir.mkdir()
    for b in range(3):
        m = io.read_triangle_mesh(os.path.join(pred, f"{b:06d}.ply"))
        p, _, _ = MR.sample_stream(np.asarray(m.vertices), np.asarray(m.triangles), n, *MESH.seed_state(5 + b))
        write_ply(str(pts_dir / f"{b:06d}.ply"), p)
    _, a = E.score_scans(seq, pred, None, 50.0, "refine", "cpu", mesh_seed=5)
    _, b = E.score_scans(seq, str(pts_dir), None, 50.0, "refine", "cpu")
    fa = E.to_json(E.fold({k: M.record_from_rows(r) for k, r in a.items()}, verbose=False))
    fb = E.to_json(E.fold({k: M.record_from_rows(r) for k, r in b.items()}, verbose=False))
    assert fa == fb
    assert all(M.record_from_rows(a[k]).n_pred < n for k in a)                  # the 50 m filter dropped the far triangle's points
    split = {}
    for rank in range(2):                                           # the samples do not depend on the rank split
        split.update(E.score_scans(seq, pred, None, 50.0, "refine", "cpu", rank=rank, world=2, mesh_seed=5)[1])
    assert all(torch.equal(split[k], a[k]) for k in a)


def test_eval_path_mesh_options():
    from click.testing import CliRunner
    res = CliRunner().invoke(E.main, ["-p", "x/", "--mesh", "--random-weights"])
    assert res.exit_code != 0 and "--mesh scores mesh files" in res.output
    res = CliRunner().invoke(E.main, ["--help"])
    assert "--mesh" in res.output and "--seed" in res.output
    assert json.dumps(E.to_json({"a": 1}))
