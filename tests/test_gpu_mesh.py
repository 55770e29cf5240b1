"""Mesh sampling on the GPU (csrc/mesh.cu through lidiff_b200.mesh) against the restatement of open3d's SamplePointsUniformly in
tests/mesh_reference.py, bit for bit: single triangles, meshes with degenerate triangles, a 1000 x 1000-vertex height field at
coordinates offset by 1e5, consecutive calls on one stream, injected words at the r >= 1 guard, bad input, and `eval_path --mesh`
end to end."""
import json
import os

import numpy as np
import pytest
import torch

import mesh_reference as MR
from lidiff_b200 import _lib
from lidiff_b200 import mesh as MESH

pytestmark = pytest.mark.gpu

UNIT = (np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), np.array([[0, 1, 2]], np.int32))


def _degenerate_mesh(n_tris=1000, seed=0):
    g = np.random.default_rng(seed)
    v = g.normal(0.0, 20.0, (600, 3))
    t = g.integers(0, 600, (n_tris, 3)).astype(np.int32)
    t[::9, 2] = t[::9, 0]                                       # repeated vertex: zero area
    v[t[5::13, 1]] = v[t[5::13, 0]]                             # coincident vertices: zero area
    return v, t


@pytest.fixture(scope="module")
def height_field():
    return MR.height_field(1000, seed=7, offset=1e5)             # 1 996 002 triangles


def _check(v, t, n, seed):
    key, pos = MESH.seed_state(seed)
    pts, key2, pos2 = MESH.sample_points_uniformly(v, t, n, key, pos)
    want, wkey, wpos = MR.sample_stream(v, t, n, key, pos)
    assert pts.shape == (n, 3) and pts.dtype == torch.float64
    got = pts.cpu().numpy()
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), f"{int((got != want).any(1).sum())} of {n} points differ"
    assert np.array_equal(key2, wkey) and pos2 == wpos
    return key2, pos2


@pytest.mark.parametrize("n", [1, 7, 1000000])
def test_single_triangle(n):
    _check(*UNIT, n, 1)
    v = np.array([[1e5 + 0.3, -2e5, 7.0], [1e5 - 4.0, -2e5 + 0.5, 7.25], [1e5 + 1.0, -2e5 + 3.0, 6.0]])
    _check(v, np.array([[2, 0, 1]]), n, 2)


@pytest.mark.parametrize("n", [1, 7, 1000000])
def test_mesh_with_degenerate_triangles(n):
    _check(*_degenerate_mesh(), n, 3)


@pytest.mark.parametrize("n", [1, 7, 1000000])
def test_height_field_of_two_million_triangles_offset_by_1e5(height_field, n):
    v, t = height_field
    assert t.shape[0] == 2 * 999 * 999
    _check(v, t, n, 4)


def test_areas_and_surface_area_bit_for_bit(height_field):
    v, t = height_field
    h = _lib.get_handle("cuda")
    vv, tt = MESH._mesh(v, t, h.device)
    area = torch.empty(t.shape[0], dtype=torch.float64, device=h.device)
    info = torch.empty(24, dtype=torch.uint8, device=h.device)
    scratch = h.mesh_sample_scratch(t.shape[0])
    h.mesh_sample_prepare(vv, tt, 1000000, area, info, scratch)
    want = MR.areas(v, t)
    assert np.array_equal(area.cpu().numpy(), want)
    rec = np.frombuffer(info.cpu().numpy().tobytes(), MESH._INFO)[0]
    assert rec["status"] == 0 and rec["surface_area"] == MR.surface_area(want) and rec["last_count"] == 1000000
    n_t = scratch[:8 * t.shape[0]].view(torch.int64).cpu().numpy()
    assert np.array_equal(n_t, MR.counts(want, 1000000))
    assert MESH.surface_area(v, t) == MR.surface_area(want)


def test_consecutive_calls_continue_the_stream():
    v, t = _degenerate_mesh(seed=1)
    key, pos = MESH.seed_state(5)
    for n in (1, 7, 155, 1000, 624, 100001):
        pts, key2, pos2 = MESH.sample_points_uniformly(v, t, n, key, pos)
        want, wkey, wpos = MR.sample_stream(v, t, n, key, pos)
        assert np.array_equal(pts.cpu().numpy(), want) and np.array_equal(key2, wkey) and pos2 == wpos
        key, pos = key2, pos2


def test_shim_global_stream_on_the_gpu():
    from lidiff_b200.shims.open3d import geometry, utility
    v, t = _degenerate_mesh(seed=2)
    utility.random.seed(8)
    m = geometry.TriangleMesh(v, t)
    a, b = (np.asarray(m.sample_points_uniformly(n).points) for n in (1000, 333))
    key, pos = MESH.seed_state(8)
    wa, key, pos = MR.sample_stream(v, t, 1000, key, pos)
    wb, key, pos = MR.sample_stream(v, t, 333, key, pos)
    assert np.array_equal(a, wa) and np.array_equal(b, wb)


@pytest.mark.parametrize("fill", ["ones", "mixed"])
def test_injected_words_exercise_the_guard(fill):
    v, t = _degenerate_mesh(seed=3)
    n = 4096
    g = np.random.default_rng(0)
    if fill == "ones":
        w = np.full(4 * n, 0xFFFFFFFF, np.uint32)
    else:
        w = g.integers(0, 2 ** 32, 4 * n, dtype=np.uint64).astype(np.uint32)
        w[0::3] = 0xFFFFFFFF                                    # hi words of all ones: r rounds to 1 when lo >= 0xFFFFFC00
        w[1::4] = 0xFFFFFFFF
        w[0:64:8] = 0xFFFFFC00                                   # lo at the rounding edge
        w[4:64:8] = 0xFFFFFBFF
        w[8:40:4] = 0
    h = _lib.get_handle("cuda")
    vv, tt = MESH._mesh(v, t, h.device)
    scratch, _ = MESH._prepare(h, vv, tt, n)
    words = torch.from_numpy(w.view(np.int32)).to(h.device)
    out = torch.empty((n, 3), dtype=torch.float64, device=h.device)
    h.mesh_sample_points(vv, tt, scratch, words, n, out)
    want = MR.sample(v, t, n, w)
    assert np.array_equal(out.cpu().numpy(), want) and np.isfinite(want).all()
    assert (MR.canonical(w[0::2], w[1::2]) == np.nextafter(1.0, 0.0)).any()


def test_bad_input_raises_before_any_sampling_launch():
    v, t = UNIT
    nan = v.copy()
    nan[2, 0] = np.inf
    h = _lib.get_handle("cuda")
    cases = [(v, t, 0, ValueError), (v, np.zeros((0, 3), np.int32), 5, ValueError), (v, np.array([[0, 1, 3]], np.int32), 5, ValueError),
             (v, np.array([[0, -7, 1]], np.int32), 5, ValueError), (nan, t, 5, ValueError),
             (v, np.array([[0, 0, 1], [1, 2, 2]], np.int32), 5, ValueError),
             (np.array([[0.0, 0, 0], [1e300, 0, 0], [0, 1e300, 0]]), t, 5, ValueError)]
    key, pos = MESH.seed_state(6)
    for v_, t_, n, exc in cases:
        l0 = h.launch_count()
        with pytest.raises(exc):
            MESH.sample_points_uniformly(v_, t_, n, key, pos)
        assert h.launch_count() - l0 <= 5                          # the prepare kernels at most: no MT words, no sampling
    _check(*_degenerate_mesh(seed=4), 1000, 6)                  # a valid call afterwards


def test_kernels_run_on_the_device():
    h = _lib.get_handle("cuda")
    l0 = h.launch_count()
    MESH.sample_points_uniformly(*UNIT, 10, *MESH.seed_state(0))
    assert h.launch_count() - l0 == 7                           # 5 prepare kernels, the MT19937 words, the sampling


def test_eval_path_mesh_end_to_end(tmp_path):
    from click.testing import CliRunner
    from eval_sequence import make_sequence
    from lidiff_b200.shims.open3d.io import read_triangle_mesh
    from lidiff_b200.tools.diff_completion_pipeline import write_ply
    from lidiff_b200.tools.eval_path import main
    from mesh_files import write_mesh_predictions
    seq, pred = make_sequence(str(tmp_path))
    write_mesh_predictions(pred)
    pts_dir = tmp_path / "points"
    pts_dir.mkdir()
    for b in range(3):
        m = read_triangle_mesh(os.path.join(pred, f"{b:06d}.ply"))
        p, _, _ = MR.sample_stream(np.asarray(m.vertices), np.asarray(m.triangles), 1000000, *MESH.seed_state(17 + b))
        write_ply(str(pts_dir / f"{b:06d}.ply"), p)
    for args in (["-p", pred + "/", "--data", seq, "--mesh", "--seed", "17"], ["-p", str(pts_dir) + "/", "--data", seq]):
        res = CliRunner().invoke(main, args, catch_exceptions=False)
        assert res.exit_code == 0, res.output
    a = json.load(open(os.path.join(pred, "res_log.yaml")))
    b = json.load(open(pts_dir / "res_log.yaml"))
    assert a == b and np.isfinite(a["cd_mean"])
