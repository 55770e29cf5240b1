"""Host-side checks of point-cloud rendering: the numpy restatement of lb2_render_splat / lb2_render_shade (render_reference.py)
against closed forms, the PNG writer, and the host logic of lidiff_b200.render, the vis_pcd CLI and the open3d shim's
draw_geometries on the CPU stand-in of tests/fake_render_backend.py."""
import importlib.util
import math
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch

import fake_render_backend
import render_reference as rr
from lidiff_b200 import render as R
from lidiff_b200.synth import synthetic_scan


def _cam(**kw):
    d = dict(lookat=(0.0, 0.0, 0.0), front=(0.0, 0.0, 1.0), up=(0.0, 1.0, 0.0), distance=10.0, width=64, height=48)
    d.update(kw)
    return R.Camera(**d)


# ---- the restatement against closed forms ------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", [(64, 48), (65, 47), (1, 1), (1920, 1080)])
def test_point_at_lookat_lands_on_the_image_centre(size):
    cam = _cam(lookat=(3.5, -2.25, 1.0), width=size[0], height=size[1])
    depth, u, v, ok = rr.project(np.array([cam.lookat]), cam)
    assert ok[0] and u[0] == size[0] / 2 and v[0] == size[1] / 2 and depth[0] == cam.distance
    cam = _cam(lookat=(3.5, -2.25, 1.0), front=(0.3, -0.2, 1.0), up=(0.1, 1.0, 0.2), width=size[0], height=size[1])
    depth, u, v, ok = rr.project(np.array([cam.lookat]), cam)      # oblique: the centre up to the rounding of d
    assert ok[0] and abs(u[0] - size[0] / 2) < 1e-9 and abs(v[0] - size[1] / 2) < 1e-9
    assert depth[0] == pytest.approx(cam.distance, rel=1e-14)


@pytest.mark.parametrize("s", range(1, 16))
def test_an_integer_point_size_covers_s_by_s_pixels(s):
    for centre in (32.0, 32.5, 31.5, 20.25, 20.75, 17.125, 40.0 + 1 / 1024):
        lo, hi = rr.span(np.array([centre]), 0.5 * s, 64)
        assert hi[0] - lo[0] == s, (centre, s)
        cols = np.arange(lo[0], hi[0])
        assert np.all(centre - 0.5 * s <= cols + 0.5) and np.all(cols + 0.5 < centre + 0.5 * s)
    cam = _cam(width=64 + (s % 2), height=48)
    keys = rr.splat(np.array([cam.lookat]), cam, s)
    hit = np.nonzero(keys != rr.EMPTY)[0]
    assert hit.shape[0] == s * s
    rows, cols = hit // cam.width, hit % cam.width
    assert rows.max() - rows.min() == s - 1 and cols.max() - cols.min() == s - 1


def test_footprint_is_clipped_at_the_image_borders():
    lo, hi = rr.span(np.array([0.0, -3.0, 64.0, 1e300, -np.inf]), 2.5, 64)
    assert list(np.maximum(hi - lo, 0)) == [2, 0, 3, 0, 0] and lo[0] == 0 and hi[2] == 64


def test_camera_basis_is_orthonormal():
    g = np.random.default_rng(0)
    for _ in range(50):
        f, u = g.normal(size=3) * 10 ** g.uniform(-3, 3), g.normal(size=3)
        F, Rt, U, _ = rr.basis(_cam(front=f, up=u))
        M = np.array([F, Rt, U])
        assert np.abs(M @ M.T - np.eye(3)).max() < 1e-14
        assert np.linalg.det(np.array([Rt, U, F])) == pytest.approx(1.0)          # right x up' = F: a right-handed frame
    F, Rt, U, eye = rr.basis(_cam())
    assert (Rt, U, F, eye) == ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (0.0, 0.0, 10.0))


def test_default_view_contains_a_scan():
    pts = synthetic_scan(0)
    cam = R.Camera.fit(pts)
    lo, hi = pts.min(0), pts.max(0)
    assert cam.lookat == tuple((lo + hi) / 2) and cam.front == (0.0, 0.0, 1.0) and cam.up == (0.0, 1.0, 0.0)
    assert cam.distance == pytest.approx(0.7 * (hi - lo).max() / math.tan(math.radians(30.0)))
    corners = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
    for p in (pts, corners):
        _, u, v, ok = rr.project(p, cam)
        assert ok.all() and (u >= 0).all() and (u < cam.width).all() and (v >= 0).all() and (v < cam.height).all()


def test_jet_ends_and_knots():
    assert tuple(rr.jet(0.0)) == (0.0, 0.0, 0.5)                # dark blue
    assert tuple(rr.jet(1.0)) == (0.5, 0.0, 0.0)                # dark red
    assert tuple(rr.jet(0.5)) == (0.5, 1.0, 0.5)
    knots = sorted({(c + k) / 2 for c in (1.5, 1.0, 0.5) for k in (-0.75, -0.25, 0.25, 0.75)})
    for t in knots:
        a, b = rr.jet(t - 1e-9), rr.jet(t + 1e-9)
        assert np.abs(a - b).max() < 1e-8, t
    t = np.linspace(-0.5, 1.5, 4001)
    assert np.abs(np.diff(rr.jet(t), axis=0)).max() <= 4 * (t[1] - t[0]) + 1e-12      # slope 2 / 0.5


def test_nearest_point_wins_and_ties_go_to_the_lower_index():
    cam = _cam()
    pts = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, 0.0, 1.0], [0.0, 0.0, -1.0]])
    keys = rr.splat(pts, cam, 3)
    hit = keys[keys != rr.EMPTY]
    assert hit.shape[0] == 9 and np.all(hit & np.uint64(0xFFFFFFFF) == 1)
    assert np.all((hit >> np.uint64(32)).astype(np.uint32).view(np.float32) == np.float32(9.0))


def test_shade_headlight_and_colours():
    cam = _cam(width=8, height=8)
    pts = np.array([[0.0, 0.0, 0.0]])
    keys = rr.splat(pts, cam, 1)
    rgb = rr.shade(keys, pts, cam, normals=np.array([[0.0, 0.0, -1.0]]), colors=np.array([[1.0, 0.5, 2.0]]))
    assert tuple(rgb[3, 3]) == (255, 128, 255) and (rgb.reshape(-1, 3).sum(1) == 765).sum() == 63
    rgb = rr.shade(keys, pts, cam, normals=np.array([[1.0, 0.0, 0.0]]), colors=np.array([[1.0, 1.0, 1.0]]))
    assert tuple(rgb[3, 3]) == (64, 64, 64)                     # rint(255 * 0.25) = 64
    rgb = rr.shade(keys, pts, cam, normals=np.array([[np.nan, 0.0, 0.0]]), colors=np.array([[0.2, np.nan, -1.0]]))
    assert tuple(rgb[3, 3]) == (51, 0, 0)


def test_heights_outside_the_z_range_take_the_colour_of_its_ends():
    cam = _cam(width=8, height=8)
    for z, colour in ((-5.0, (0, 0, 128)), (0.0, (0, 0, 128)), (1.0, (128, 0, 0)), (7.0, (128, 0, 0))):
        pts = np.array([[0.0, 0.0, z]])
        rgb = rr.shade(rr.splat(pts, cam, 1), pts, cam, z_lo=0.0, z_hi=1.0)
        assert tuple(rgb[3, 3]) == colour, z


# ---- PNG -----------------------------------------------------------------------------------------------------------------------
def _parse_png(data):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(kind + body) & 0xFFFFFFFF, kind
        chunks.append((kind, body))
        pos += 12 + n
    return chunks


def decode_png(data):
    chunks = _parse_png(data)
    assert [k for k, _ in chunks][0] == b"IHDR" and chunks[-1] == (b"IEND", b"")
    w, h, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", chunks[0][1])
    assert (depth, ctype, comp, filt, inter) == (8, 2, 0, 0, 0)
    raw = zlib.decompress(b"".join(b for k, b in chunks if k == b"IDAT"))
    rows = np.frombuffer(raw, np.uint8).reshape(h, 1 + 3 * w)
    assert np.all(rows[:, 0] == 0)
    return rows[:, 1:].reshape(h, w, 3)


@pytest.mark.parametrize("shape", [(1, 1), (3, 5), (480, 640)])
def test_png_round_trip(tmp_path, shape):
    img = np.random.default_rng(1).integers(0, 256, shape + (3,), dtype=np.uint8)
    path = R.write_png(str(tmp_path / "sub" / "a.png"), torch.from_numpy(img))
    assert np.array_equal(decode_png(open(path, "rb").read()), img)


@pytest.mark.parametrize("bad", [np.zeros((2, 2), np.uint8), np.zeros((2, 2, 3), np.float32), np.zeros((0, 4, 3), np.uint8)])
def test_png_refuses_what_is_not_an_rgb_image(tmp_path, bad):
    with pytest.raises(ValueError):
        R.write_png(str(tmp_path / "a.png"), bad)


# ---- lidiff_b200.render on the CPU stand-in ------------------------------------------------------------------------------------
def test_render_matches_the_restatement_on_the_stand_in(monkeypatch):
    h = fake_render_backend.install(monkeypatch)
    pts = synthetic_scan(0)[::40]
    cam = R.Camera.fit(pts, width=160, height=90)
    nrm = np.random.default_rng(2).normal(size=pts.shape)
    rgb = R.render(pts, cam, normals=nrm, point_size=2)
    _, ref = rr.render(pts, cam, normals=nrm, point_size=2)
    assert rgb.dtype == torch.uint8 and np.array_equal(rgb.numpy(), ref) and h.launches == 2
    assert (ref != 255).any()


def test_render_of_no_points_is_white(monkeypatch):
    fake_render_backend.install(monkeypatch)
    rgb = R.render(np.zeros((0, 3)), _cam(width=7, height=3))
    assert rgb.shape == (3, 7, 3) and bool((rgb == 255).all())


@pytest.mark.parametrize("case", ["shape", "point_size", "normals", "colors", "colors_rgba", "normals_flat", "z_range", "camera"])
def test_render_rejects_bad_input(monkeypatch, case):
    fake_render_backend.install(monkeypatch)
    pts, kw = np.zeros((4, 3)), {}
    if case == "shape":
        pts = np.zeros((4, 2))
    elif case == "point_size":
        kw = {"point_size": 0}
    elif case == "normals":
        kw = {"normals": np.zeros((3, 3))}
    elif case == "colors":
        kw = {"colors": np.zeros((5, 3))}
    elif case == "colors_rgba":
        kw = {"colors": np.zeros((4, 4))}
    elif case == "normals_flat":
        kw = {"normals": np.zeros(12)}
    elif case == "z_range":
        kw = {"z_range": (1.0, 0.0)}
    with pytest.raises(ValueError):
        R.render(pts, "not a camera" if case == "camera" else _cam(), **kw)


@pytest.mark.parametrize("kw", [{"width": 0}, {"height": -2}, {"width": 2.5}, {"front": (0, 0, 0)}, {"up": (0, 0, 0)},
                                {"up": (0, 0, 3)}, {"distance": 0.0}, {"distance": float("inf")}, {"lookat": (0, np.nan, 0)},
                                {"fov": 180}])
def test_camera_rejects_bad_values(kw):
    with pytest.raises(ValueError):
        _cam(**kw)


def test_camera_fit_overrides_and_degenerate_clouds():
    cam = R.Camera.fit(np.array([[1.0, 2.0, 3.0], [np.nan, 0, 0]]), front=(1, 0, 0), up=(0, 0, 1), zoom=1.0, width=10, height=20)
    assert cam.lookat == (1.0, 2.0, 3.0) and cam.front == (1.0, 0.0, 0.0) and cam.up == (0.0, 0.0, 1.0)
    assert cam.distance == pytest.approx(1.0 / math.tan(math.radians(30.0))) and cam.focal == pytest.approx(10.0 / math.tan(math.radians(30)))
    assert R.Camera.fit(np.zeros((0, 3))).lookat == (0.5, 0.5, 0.5)
    with pytest.raises(ValueError):
        R.Camera.fit(np.zeros((3, 3)), zoom=0)


# ---- the CLI and the shim on the stand-in -----------------------------------------------------------------------------------
def _write_cloud(path, pts):
    from lidiff_b200.tools.diff_completion_pipeline import write_ply
    if path.endswith(".bin"):
        np.concatenate([pts, np.zeros((pts.shape[0], 1))], 1).astype(np.float32).tofile(path)
    else:
        write_ply(path, pts)


def test_vis_pcd_cli_writes_the_reference_filtered_view(monkeypatch, tmp_path):
    from click.testing import CliRunner
    from lidiff_b200.tools import vis_pcd
    fake_render_backend.install(monkeypatch)
    pts = synthetic_scan(0)[::97]
    pts = np.concatenate([pts, [[60.0, 0.0, 0.0], [1.0, 1.0, 3.5], [1.0, 1.0, -2.6]]])
    _write_cloud(str(tmp_path / "a.ply"), pts)
    out = tmp_path / "v.png"
    r = CliRunner().invoke(vis_pcd.main, ["-p", str(tmp_path / "a.ply"), "--out", str(out), "--width", "96", "--height", "64",
                                          "--point-size", "3"])
    assert r.exit_code == 0, r.output
    kept = vis_pcd.radius_filter(pts, 50.0)
    assert kept.shape[0] == pts.shape[0] - 3
    from lidiff_b200.normals import estimate_normals
    cam = R.Camera.fit(kept, width=96, height=64)
    _, ref = rr.render(kept, cam, normals=estimate_normals(kept, knn=30).numpy(), point_size=3)
    assert np.array_equal(decode_png(out.read_bytes()), ref)


def test_vis_pcd_cli_renders_every_cloud_of_a_directory(monkeypatch, tmp_path):
    from click.testing import CliRunner
    from lidiff_b200.tools import vis_pcd
    fake_render_backend.install(monkeypatch)
    d = tmp_path / "refine"
    d.mkdir()
    _write_cloud(str(d / "000001.ply"), synthetic_scan(0)[::301])
    _write_cloud(str(d / "000002.bin"), synthetic_scan(1)[::301])
    (d / "notes.txt").write_text("x")
    r = CliRunner().invoke(vis_pcd.main, ["-p", str(d), "--out", str(tmp_path / "views" / "x.png"), "--width", "32", "--height", "24",
                                          "--front", "1", "0", "1", "--zoom", "0.5"])
    assert r.exit_code == 0, r.output
    assert sorted(os.listdir(tmp_path / "views")) == ["000001.png", "000002.png"]
    r = CliRunner().invoke(vis_pcd.main, ["-p", str(tmp_path / "missing.ply")])
    assert r.exit_code != 0 and "no such point cloud" in r.output
    r = CliRunner().invoke(vis_pcd.main, ["-p", str(d / "000001.ply"), "--out", str(tmp_path / "y.png"), "--width", "0"])
    assert r.exit_code != 0 and "width" in r.output


@pytest.fixture
def o3d(monkeypatch):
    import lidiff_b200.shims as sh
    sh.install()
    sys.modules.pop("open3d", None)
    for k in [k for k in sys.modules if k.startswith("open3d.")]:
        monkeypatch.delitem(sys.modules, k)
    import open3d
    return open3d


def test_shim_draw_geometries_writes_numbered_pngs(monkeypatch, tmp_path, o3d):
    fake_render_backend.install(monkeypatch)
    monkeypatch.setenv("LB2_O3D_RENDER_DIR", str(tmp_path))
    pts = synthetic_scan(0)[::500]
    pcd = o3d.geometry.PointCloud(o3d.utility.Vector3dVector(pts))
    assert pcd.paint_uniform_color([1.0, 0.0, 0.0]) is pcd and np.asarray(pcd.colors).shape == pts.shape
    p0 = o3d.visualization.draw_geometries([pcd], window_name="scan", width=40, height=30)
    p1 = o3d.visualization.draw_geometries([pcd], window_name="scan", width=40, height=30, front=[0, 1, 1], up=[0, 0, 1], zoom=0.3)
    assert [os.path.basename(p0), os.path.basename(p1)] == ["scan_0.png", "scan_1.png"]
    img = decode_png(open(p0, "rb").read())
    _, ref = rr.render(pts, R.Camera.fit(pts, width=40, height=30), colors=np.asarray(pcd.colors))
    assert np.array_equal(img, ref)
    assert set(map(tuple, img.reshape(-1, 3))) == {(255, 255, 255), (255, 0, 0)}


@pytest.mark.parametrize("kw", [{"point_show_normal": True}, {"mesh_show_wireframe": True}, {"mesh_show_back_face": True}])
def test_shim_draw_geometries_refuses_what_it_does_not_draw(monkeypatch, tmp_path, o3d, kw):
    fake_render_backend.install(monkeypatch)
    monkeypatch.setenv("LB2_O3D_RENDER_DIR", str(tmp_path))
    pcd = o3d.geometry.PointCloud(o3d.utility.Vector3dVector(np.zeros((3, 3))))
    with pytest.raises(NotImplementedError):
        o3d.visualization.draw_geometries([pcd], **kw)
    with pytest.raises(NotImplementedError):
        o3d.visualization.draw_geometries([o3d.geometry.VoxelGrid()])
    assert os.listdir(tmp_path) == []


REF = os.environ.get("LIDIFF_REFERENCE_DIR", "")


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "lidiff", "vis_pcd.py")),
                    reason="LIDIFF_REFERENCE_DIR (a reference checkout) is not set")
def test_reference_vis_pcd_writes_a_png_on_the_shims(monkeypatch, tmp_path, o3d):
    from click.testing import CliRunner
    fake_render_backend.install(monkeypatch)
    monkeypatch.setenv("LB2_O3D_RENDER_DIR", str(tmp_path))
    _write_cloud(str(tmp_path / "c.ply"), synthetic_scan(0)[::200])
    spec = importlib.util.spec_from_file_location("ref_vis_pcd", os.path.join(REF, "lidiff", "vis_pcd.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.o3d is o3d
    r = CliRunner().invoke(mod.main, ["-p", str(tmp_path / "c.ply"), "-r", "50"])
    assert r.exit_code == 0, r.output
    assert os.path.isfile(tmp_path / "Open3D_0.png")
    assert decode_png((tmp_path / "Open3D_0.png").read_bytes()).shape == (1080, 1920, 3)


def test_vis_pcd_names_clouds_that_share_a_stem_apart(monkeypatch, tmp_path):
    from click.testing import CliRunner
    from lidiff_b200.tools import vis_pcd
    fake_render_backend.install(monkeypatch)
    assert vis_pcd.png_names(["d/a.bin", "d/a.ply", "d/b.ply"]) == ["a.bin.png", "a.ply.png", "b.png"]
    d = tmp_path / "c"
    d.mkdir()
    _write_cloud(str(d / "x.ply"), synthetic_scan(0)[::301])
    _write_cloud(str(d / "x.bin"), synthetic_scan(1)[::301])
    r = CliRunner().invoke(vis_pcd.main, ["-p", str(d), "--out", str(tmp_path / "v" / "o.png"), "--width", "16", "--height", "8"])
    assert r.exit_code == 0, r.output
    assert sorted(os.listdir(tmp_path / "v")) == ["x.bin.png", "x.ply.png"]


# ---- vis_steps: argument handling ---------------------------------------------------------------------------------------------
def test_vis_steps_parses_steps():
    from lidiff_b200.tools.vis_steps import parse_steps
    assert parse_steps("0,10,25,50", 50) == [0, 10, 25, 50]
    assert parse_steps("50, 0,25,25", 50) == [0, 25, 50]
    assert parse_steps(None, 50) == [0, 10, 25, 50] and parse_steps("", 5) == [0, 1, 2, 5] and parse_steps(None, 1) == [0, 1]
    for bad in ("0,51", "-1,3", "a,b", ",", "1.5"):
        with pytest.raises(ValueError):
            parse_steps(bad, 50)


@pytest.mark.parametrize("args, msg", [([], "--random-weights"), (["-d", "a.ckpt"], "--random-weights"),
                                       (["--random-weights", "--steps", "0,60"], "outside"),
                                       (["--random-weights", "-T", "5", "--steps", "x"], "integers"),
                                       (["--random-weights", "-T", "0"], "-T")])
def test_vis_steps_refuses_bad_arguments_before_any_work(tmp_path, args, msg):
    from click.testing import CliRunner
    from lidiff_b200.tools import vis_steps
    scan = tmp_path / "s.bin"
    _write_cloud(str(scan), synthetic_scan(0)[::100])
    r = CliRunner().invoke(vis_steps.main, ["--scan", str(scan), "--out", str(tmp_path / "o.png")] + args)
    assert r.exit_code == 2 and msg in r.output, r.output
    assert not (tmp_path / "o.png").exists()


def test_vis_steps_strip_puts_the_panels_side_by_side(monkeypatch):
    from lidiff_b200.tools import vis_steps
    fake_render_backend.install(monkeypatch)
    a, b = synthetic_scan(0)[::200], synthetic_scan(1)[::200]
    traj = {"scan": torch.from_numpy(a), "steps": {5: torch.from_numpy(b), 0: torch.from_numpy(b[::2])},
            "post": torch.from_numpy(a[::3]), "refined": torch.from_numpy(b[::3])}
    panels = vis_steps.panels_of(traj)
    assert [p.shape[0] for p in panels] == [a.shape[0], b[::2].shape[0], b.shape[0], a[::3].shape[0], b[::3].shape[0]]
    cam = R.Camera.fit(a, width=24, height=16)
    img = vis_steps.strip(panels, cam, (float(a[:, 2].min()), float(a[:, 2].max())), 2.0).numpy()
    assert img.shape == (16, 5 * 24, 3)
    _, ref = rr.render(b, cam, point_size=2.0, z_range=(float(a[:, 2].min()), float(a[:, 2].max())))
    assert np.array_equal(img[:, 2 * 24:3 * 24], ref)
