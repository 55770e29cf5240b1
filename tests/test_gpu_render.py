"""lb2_render_splat / lb2_render_shade on the GPU against the numpy restatement of tests/render_reference.py, bit for bit: the
z-buffer keys (so the depth and the winning index of every pixel) and the RGB bytes, on scans, a refined-sized cloud, ties,
points at and behind the near rule and across the image borders, non-finite rows and normals, coloured clouds, 1x1 and 4096x4096
images and point sizes 1 to 15."""
import numpy as np
import pytest
import torch

import render_reference as rr
from lidiff_b200 import _lib
from lidiff_b200 import render as R
from lidiff_b200.synth import synthetic_scan

pytestmark = pytest.mark.gpu


def _gpu(pts, cam, normals=None, colors=None, point_size=5.0, z_range=None):
    """(keys uint64, rgb uint8) from the device, and render()'s image (which must be the same)"""
    h = _lib.get_handle("cuda:0")
    p = torch.as_tensor(np.asarray(pts, np.float64)).cuda().contiguous()
    nrm = None if normals is None else torch.as_tensor(np.asarray(normals, np.float64)).cuda().contiguous()
    col = None if colors is None else torch.as_tensor(np.asarray(colors, np.float64)).cuda().contiguous()
    if z_range is None:
        fin = p[torch.isfinite(p).all(1)]
        z_range = (float(fin[:, 2].min()), float(fin[:, 2].max())) if fin.shape[0] else (0.0, 0.0)
    keys = torch.full((cam.height * cam.width,), -1, dtype=torch.int64, device="cuda:0")
    c = cam.c_struct()
    if p.shape[0]:
        h.render_splat(p, c, point_size, keys)
    rgb = torch.empty((cam.height, cam.width, 3), dtype=torch.uint8, device="cuda:0")
    h.render_shade(keys, p, nrm, col, z_range[0], z_range[1], c, rgb)
    via_api = R.render(p, cam, normals=nrm, colors=col, point_size=point_size, z_range=z_range)
    torch.cuda.synchronize()
    assert torch.equal(via_api, rgb), "render() differs from the two calls it makes"
    return keys.cpu().numpy().view(np.uint64), rgb.cpu().numpy()


def _check(pts, cam, normals=None, colors=None, point_size=5.0, z_range=None):
    keys, rgb = _gpu(pts, cam, normals, colors, point_size, z_range)
    ref_keys = rr.splat(pts, cam, point_size)
    if z_range is None:
        fin = np.asarray(pts)[np.isfinite(pts).all(1)]
        z_range = (float(fin[:, 2].min()), float(fin[:, 2].max())) if fin.shape[0] else (0.0, 0.0)
    ref_rgb = rr.shade(ref_keys, pts, cam, normals, colors, *z_range)
    bad = np.nonzero(keys != ref_keys)[0]
    assert bad.shape[0] == 0, f"{bad.shape[0]} keys differ, first at pixel {bad[:4]}: {keys[bad[:4]]} vs {ref_keys[bad[:4]]}"
    assert np.array_equal(rgb, ref_rgb), f"{int((rgb != ref_rgb).any(2).sum())} pixels differ"
    return keys, rgb


def _normals(pts):
    from lidiff_b200.normals import estimate_normals
    return estimate_normals(pts, knn=30).cpu().numpy()


@pytest.mark.parametrize("s", [1, 2, 5, 15])
def test_scan_default_camera(s):
    pts = synthetic_scan(0)
    keys, rgb = _check(pts, R.Camera.fit(pts), normals=_normals(pts), point_size=s)
    assert (keys != rr.EMPTY).mean() > 0.01 and (rgb != 255).any()


@pytest.mark.parametrize("s", [1, 3.7])
def test_scan_oblique_camera(s):
    pts = synthetic_scan(3)
    cam = R.Camera.fit(pts, front=(0.4, -0.7, 0.35), up=(0.0, 0.0, 1.0), zoom=0.35, width=1280, height=720, fov=45)
    _check(pts, cam, normals=_normals(pts), point_size=s)


def test_refined_sized_cloud():
    from normals_oracle import refined_like
    pts = refined_like(0)
    assert pts.shape[0] == 1_020_000
    _check(pts, R.Camera.fit(pts), normals=_normals(pts), point_size=5)


def test_identical_points_tie_to_the_lowest_index():
    pts = np.tile(np.array([[1.25, -0.5, 0.75]]), (100_000, 1))
    pts[:7] = np.nan
    cam = R.Camera.fit(pts, width=64, height=64)
    keys, _ = _check(pts, cam, point_size=5)
    hit = keys[keys != rr.EMPTY]
    assert hit.shape[0] == 25 and np.all(hit & np.uint64(0xFFFFFFFF) == 7)


def test_behind_near_and_across_the_borders():
    cam = R.Camera(lookat=(0.0, 0.0, 0.0), front=(0.0, 0.0, 1.0), up=(0.0, 1.0, 0.0), distance=10.0, width=200, height=100)
    g = np.random.default_rng(4)
    near = 1e-3 * cam.distance
    eye_z = cam.distance
    rows = [[0.0, 0.0, eye_z - near], [0.0, 0.0, np.nextafter(eye_z - near, -np.inf)], [0.0, 0.0, eye_z + 1.0], [0.0, 0.0, eye_z],
            [0.01, 0.0, eye_z - 2 * near], [0.0, 0.0, -1e300], [1e300, 1e300, 0.0], [-1e308, 1e308, -1e308]]
    # points whose squares straddle each border: x_c / depth = (u - W/2) / f with u near 0 and W, likewise v
    f = cam.focal
    for u in (0.0, 0.3, -0.2, 200.0, 199.6, 201.1):
        for v in (50.0, 0.0, 0.4, -0.45, 100.0, 99.7):
            rows.append([(u - 100.0) / f * 10.0, -(v - 50.0) / f * 10.0, 0.0])
    rows += list(np.column_stack([g.uniform(-12, 12, 2000), g.uniform(-7, 7, 2000), g.uniform(-15, 9.99, 2000)]))
    pts = np.array(rows, np.float64)
    for s in (1, 2, 5, 15):
        _check(pts, cam, point_size=s)


def test_non_finite_rows_and_normals():
    pts = synthetic_scan(1)[::7].copy()
    g = np.random.default_rng(5)
    bad = g.choice(pts.shape[0], 500, replace=False)
    pts[bad[:200], g.integers(0, 3, 200)] = np.nan
    pts[bad[200:350], 0] = np.inf
    pts[bad[350:], 2] = -np.inf
    nrm = _normals(pts)
    nrm[g.choice(pts.shape[0], 300, replace=False)] = np.nan
    nrm[:50] = np.inf
    assert np.isnan(nrm).any(1).sum() >= 300
    _check(pts, R.Camera.fit(pts), normals=nrm, point_size=3)


def test_coloured_cloud():
    pts = synthetic_scan(2)[::3]
    g = np.random.default_rng(6)
    col = g.uniform(-0.2, 1.2, pts.shape)
    col[:20] = np.nan
    _check(pts, R.Camera.fit(pts, width=800, height=600), normals=_normals(pts), colors=col, point_size=2)
    _check(pts, R.Camera.fit(pts, width=800, height=600), colors=np.full(pts.shape, 0.5), point_size=2)


@pytest.mark.parametrize("size", [(1, 1), (4096, 4096)])
def test_extreme_image_sizes(size):
    pts = synthetic_scan(0)[::2]
    cam = R.Camera.fit(pts, width=size[0], height=size[1])
    _check(pts, cam, normals=_normals(pts), point_size=15 if size[0] == 1 else 2)


def test_no_points_and_a_flat_z_range():
    cam = R.Camera.fit(np.zeros((0, 3)), width=33, height=17)
    rgb = R.render(np.zeros((0, 3)), cam)
    assert rgb.shape == (17, 33, 3) and bool((rgb == 255).all())
    pts = np.array([[0.0, 0.0, 1.0], [0.5, 0.5, 1.0]])
    _, img = _check(pts, R.Camera.fit(pts, width=33, height=17), point_size=4)
    assert {tuple(p) for p in img.reshape(-1, 3)} == {(255, 255, 255), (0, 0, 128)}      # jet(0)


def test_two_runs_give_identical_bytes():
    from normals_oracle import refined_like
    pts = refined_like(1, n_base=60_000)
    cam = R.Camera.fit(pts)
    nrm = _normals(pts)
    a = R.render(pts, cam, normals=nrm, point_size=5).cpu().numpy()
    b = R.render(pts, cam, normals=nrm, point_size=5).cpu().numpy()
    assert np.array_equal(a, b) and R.encode_png(a) == R.encode_png(b)
