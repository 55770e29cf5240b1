"""The ground-truth-map kernels (lb2_map_scan / lb2_map_rehash) and lidiff_b200.maps on the GPU: bit-exact against a numpy restatement
of the documented arithmetic (tests/fake_maps_backend.py) for both division modes, streaming = one shot, growth, determinism, edge
cases, the map_from_scans CLI and the reference's recorded maps (tests/golden/map_reference.npz, recorded by
tests/golden/make_map_goldens.py)."""
import os
import sys

import numpy as np
import pytest
import torch
from click.testing import CliRunner

from fake_maps_backend import restate_map
from lidiff_b200.maps import MapBuilder

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_map_goldens as G  # noqa: E402

pytestmark = pytest.mark.gpu

VS = 0.1


def _pose(b):
    return G.lidar_pose(b, turn=0.3, step=(-3.0, 1.7, -0.2))


def _tricky_scan(g, b, n=40_000):
    """points on voxel faces (multiples of the voxel size, in the map frame for the identity pose), exactly at the 3.5 m boundary,
    negative coordinates, duplicates, remission that decides the range filter, every excluded class and upper label bits"""
    faces = (g.integers(-400, 400, (n // 4, 3)) * np.float32(VS)).astype(np.float32)
    faces = np.concatenate([faces, np.nextafter(faces, np.float32(np.inf)), np.nextafter(faces, -np.float32(np.inf))])
    quarters = (g.integers(-800, 800, (n // 8, 3)) * 0.25).astype(np.float32)           # exact multiples of 0.25 (binary)
    xyz = np.concatenate([faces, quarters, g.uniform(-30, 30, (n // 4, 3)).astype(np.float32)])
    rem = g.uniform(0, 1, (xyz.shape[0], 1)).astype(np.float32)
    b35 = np.float32(3.5)
    edge = np.array([[b35, 0, 0, 0], [0, -b35, 0, 0], [0, 0, b35, 0], [0, 0, 0, b35], [np.nextafter(b35, np.float32(4)), 0, 0, 0],
                     [np.nextafter(b35, np.float32(0)), 0, 0, 0], [2.0, 2.0, 2.0, 0.5], [3.0, 0, 0, 1.9], [3.0, 0, 0, 1.8],
                     [0, 0, 0, 3.6], [-0.05, -0.05, -0.05, 4.0], [0.05, 0.05, 0.05, 4.0]], np.float32)
    pts = np.concatenate([np.concatenate([xyz, rem], 1), edge])
    pts = np.concatenate([pts, pts[g.choice(pts.shape[0], pts.shape[0] // 5)]]).astype(np.float32)
    pts = pts[g.permutation(pts.shape[0])]
    cls = np.where(g.uniform(size=pts.shape[0]) < 0.3, g.choice(G.EXCLUDED, pts.shape[0]), g.choice(G.KEPT, pts.shape[0]))
    lab = (cls.astype(np.uint32) | (g.integers(0, 1 << 16, pts.shape[0]).astype(np.uint32) << 16)).astype(np.uint32)
    return pts, lab


def _scans(seed=0, n_scans=4, identity_first=True):
    g = np.random.default_rng(seed)
    out = []
    for b in range(n_scans):
        pts, lab = _tricky_scan(g, b)
        pose = np.eye(4) if (identity_first and b == 0) else _pose(b)
        out.append((pts, lab, pose))
    out.append((out[0][0][:5000], out[0][1][:5000], _pose(1)))                 # a scan seen again under another pose
    out.append((out[1][0], out[1][1], out[1][2]))                                # and under the same one (all duplicates)
    return out


def _build(scans, div_mode=1, **kw):
    mb = MapBuilder(VS, div_mode, "cuda", **kw)
    for pts, lab, pose in scans:
        mb.add_scan(pts, lab, pose)
    return mb


def _p12(pose):
    return np.asarray(pose)[:3, :4].astype(np.float32).reshape(-1)


@pytest.mark.parametrize("div_mode", [0, 1])
def test_bit_exact_against_the_restatement(div_mode):
    scans = _scans()
    got = _build(scans, div_mode).points().cpu().numpy()
    want = restate_map([(p, l, _p12(q)) for p, l, q in scans], VS, div_mode)
    assert got.shape == want.shape and got.shape[0] > 50_000
    assert got.tobytes() == want.tobytes()


def test_division_modes_differ_somewhere_on_faces():
    scans = _scans(1)[:1]
    a, b = (restate_map([(p, l, _p12(q)) for p, l, q in scans], VS, m) for m in (0, 1))
    assert a.shape != b.shape or a.tobytes() != b.tobytes()          # the data does reach the points where the two modes disagree


def test_streaming_equals_one_shot():
    g = np.random.default_rng(3)
    parts = [_tricky_scan(g, b, 20_000) for b in range(5)]
    pose = _pose(2)
    streamed = _build([(p, l, pose) for p, l in parts]).points().cpu().numpy()
    one = _build([(np.concatenate([p for p, _ in parts]), np.concatenate([l for _, l in parts]), pose)]).points().cpu().numpy()
    assert streamed.tobytes() == one.tobytes()


def test_growth_gives_the_same_bits():
    scans = _scans(4)
    small = _build(scans, initial_capacity=1)
    big = _build(scans, initial_capacity=1 << 22)
    assert small.rehashes >= 3 and big.rehashes == 0 and small._map.shape[0] < big._map.shape[0]
    assert small.points().cpu().numpy().tobytes() == big.points().cpu().numpy().tobytes()


def test_two_runs_give_identical_bytes():
    from lidiff_b200.synth import synthetic_scan
    g = np.random.default_rng(5)
    scans = []
    for b in range(6):
        xyz = synthetic_scan(b)
        pts = np.concatenate([xyz, g.uniform(0, 1, (xyz.shape[0], 1))], 1).astype(np.float32)
        pts = np.concatenate([pts, pts[::3]])                                  # heavy contention on the same voxels
        scans.append((pts, None, G.lidar_pose(b)))
    a, b = _build(scans).points().cpu().numpy(), _build(scans).points().cpu().numpy()
    assert a.shape[0] > 100_000 and a.tobytes() == b.tobytes()
    assert a.tobytes() == restate_map([(p, None, _p12(q)) for p, _, q in scans], VS, 1).tobytes()


def test_empty_and_fully_filtered_scans_leave_the_map_unchanged():
    scans = _scans(6)[:2]
    mb = _build(scans)
    before = mb.points().cpu().numpy().copy()
    assert mb.add_scan(np.zeros((0, 4), np.float32), np.zeros(0, np.uint32), _pose(3)) == 0
    near = np.random.default_rng(0).uniform(-1, 1, (1000, 4)).astype(np.float32)           # all within 3.5 m
    assert mb.add_scan(near, None, _pose(3)) == 0
    pts, lab = scans[0][0], np.full(scans[0][0].shape[0], 252, np.uint32)                   # all moving
    assert mb.add_scan(pts, lab, _pose(3)) == 0
    assert mb.points().cpu().numpy().tobytes() == before.tobytes()


def test_out_of_range_key_raises():
    mb = MapBuilder(VS, 1, "cuda")
    far = np.array([[4.0, 0, 0, 0], [0, 0, -(2.0 ** 20) * VS - 1.0, 0]], np.float32)
    with pytest.raises(ValueError, match="key range"):
        mb.add_scan(far)
    ok = MapBuilder(VS, 1, "cuda")
    inside = np.array([[(2.0 ** 20 - 2) * VS, 0, 0, 0]], np.float32)
    assert ok.add_scan(inside) == 1


def test_cli_end_to_end(tmp_path):
    from lidiff_b200 import kitti
    from lidiff_b200.tools import map_from_scans as MS
    for i, seq in enumerate(["00", "01"]):
        G.write_sequence(str(tmp_path / seq), n_scans=4, seed=20 + i, beams=32, azimuths=1024, margin=0)
    res = CliRunner().invoke(MS.main, ["-p", str(tmp_path), "--sequences", "00,01"], catch_exceptions=False)
    assert res.exit_code == 0, res.output
    for seq in ("00", "01"):
        got = np.load(tmp_path / seq / "map_clean.npy")
        scans = [(kitti.read_scan(p), kitti.read_labels(kitti.label_path(p)), _p12(q)) for q, p in MS.sequence_scans(str(tmp_path / seq))]
        assert got.dtype == np.float32 and got.tobytes() == restate_map(scans, VS, 1).tobytes()


def test_against_the_reference_golden(tmp_path):
    from lidiff_b200.tools import map_from_scans as MS
    ref = np.load(os.path.join(HERE, "golden", "map_reference.npz"))
    G.make_dataset(str(tmp_path), int(ref["seed"]))
    res = CliRunner().invoke(MS.main, ["-p", str(tmp_path), "-v", str(float(ref["voxel_size"])), "--div-mode", "0"],
                             catch_exceptions=False)
    assert res.exit_code == 0, res.output
    for seq in G.SEQUENCES:
        got, want = np.load(tmp_path / seq / "map_clean.npy"), ref[f"seq{seq}"]
        assert got.shape == want.shape, seq
        assert np.abs(got - want).max() <= 1e-5, seq
