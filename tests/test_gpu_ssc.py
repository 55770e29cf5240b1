"""Scene-completion grids on the GPU (csrc/ssc.cu through lidiff_b200.ssc) against the numpy restatement of tests/ssc_reference.py,
bit for bit: empty, one-voxel, random and full grids of both kinds, batches across chunk boundaries and reruns, voxelization of a
1 M-point cloud with out-of-extent and non-finite rows, confusion counts with and without invalid masks, and `eval_path --voxels`
and `--ssc` end to end."""
import json
import os

import numpy as np
import pytest
import torch

import ssc_reference as SR
from lidiff_b200 import _lib
from lidiff_b200 import ssc as S

pytestmark = pytest.mark.gpu


def _grids(kind, seed=0):
    """{name: grid} of `kind`: empty, one voxel (first, last and inside), random at several densities, full"""
    g = np.random.default_rng(seed)
    labs = {"empty": np.zeros(S.N_VOXELS, np.uint16), "full": np.full(S.N_VOXELS, 3, np.uint16)}
    for v in (0, 31, 32, 123457, S.N_VOXELS - 1):
        labs[f"one_{v}"] = np.zeros(S.N_VOXELS, np.uint16)
        labs[f"one_{v}"][v] = 40
    for d in (1e-5, 0.01, 0.3, 0.97):
        labs[f"random_{d}"] = SR.random_labels(g, d, 0.02)
    labs["all_ignored"] = np.full(S.N_VOXELS, 255, np.uint16)
    if kind == "labels":
        return labs
    return {k: SR.pack(SR.occupied(v)) for k, v in labs.items()}


@pytest.mark.parametrize("kind", ["labels", "bits"])
def test_grid_points_single_grids(kind):
    for name, grid in _grids(kind).items():
        occ = SR.occupied(grid) if kind == "labels" else SR.unpack(grid)
        pts, off = S.grid_points(grid, kind)
        want = SR.centres(occ)
        assert pts.dtype == torch.float64 and list(off) == [0, want.shape[0]], name
        assert np.array_equal(pts.cpu().numpy().view(np.uint64), want.view(np.uint64)), name
    assert S.grid_points(_grids(kind)["full"], kind)[0].shape == (S.N_VOXELS, 3)


@pytest.mark.parametrize("kind", ["labels", "bits"])
def test_grid_points_batches_and_reruns(kind):
    g = np.random.default_rng(1)
    base = list(_grids(kind, seed=2).values())
    grids = [base[i] for i in g.integers(0, len(base), S.CHUNK + 9)]     # two chunks, different counts per grid
    occ = [SR.occupied(x) if kind == "labels" else SR.unpack(x) for x in grids]
    want = [SR.centres(o) for o in occ]
    h = _lib.get_handle("cuda")
    l0 = h.launch_count()
    pts, off = S.grid_points(grids, kind)
    assert h.launch_count() - l0 == 2 * 4                                # four launches per chunk
    assert np.array_equal(np.diff(off), [w.shape[0] for w in want])
    assert np.array_equal(pts.cpu().numpy(), np.concatenate(want))
    again, off2 = S.grid_points(np.stack(grids), kind)
    assert np.array_equal(off, off2) and torch.equal(pts.view(torch.int64), again.view(torch.int64))


def test_voxelize_a_million_points_with_dropped_rows():
    g = np.random.default_rng(3)
    pts = g.uniform([-10, -35, -5], [60, 35, 8], (1_000_000, 3))
    pts[::997] = np.nan
    pts[5::1009, 1] = np.inf
    pts[7::1013, 2] = -np.inf
    pts[11::101] = [0.0, -25.6, -2.0]
    pts[13::103] = [-0.0, -0.0, -0.0]
    pts[17::107] = [51.2, 3.0, 1.0]
    pts[19::109] = [np.nextafter(51.2, 0), np.nextafter(25.6, 0), np.nextafter(4.4, 0)]
    want, nf, out = SR.voxelize(pts)
    for src in (pts, torch.from_numpy(pts).cuda()):
        bits, dropped = S.voxelize(src)
        assert np.array_equal(bits.cpu().numpy().view(np.uint32), want) and list(dropped) == [nf, out]
    assert nf > 2000 and out > 100000
    clouds = [pts[:0], pts[:1], pts[1:400000], pts[400000:400001], pts[400001:]]
    off = np.cumsum([0] + [c.shape[0] for c in clouds])
    bits, dropped = S.voxelize(pts, off)
    for k, c in enumerate(clouds):
        w, a, b = SR.voxelize(c)
        assert np.array_equal(bits[k].cpu().numpy().view(np.uint32), w) and list(dropped[k]) == [a, b], k


def test_round_trips_on_the_device():
    g = np.random.default_rng(4)
    lab = SR.random_labels(g, 0.05, 0.05)
    pts, _ = S.grid_points(lab, "labels")
    bits, dropped = S.voxelize(pts)
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), SR.pack(SR.occupied(lab))) and list(dropped) == [0, 0]
    again, _ = S.grid_points(bits, "bits")
    assert torch.equal(again, pts)


def test_confusion_counts():
    g = np.random.default_rng(5)
    labs = [SR.random_labels(g, d, 0.05) for d in (0.0, 0.001, 0.1, 0.6)] + [np.full(S.N_VOXELS, 255, np.uint16)]
    preds = [SR.pack(g.random(S.N_VOXELS) < d) for d in (0.5, 0.001, 0.12, 0.0, 1.0)]
    invs = [SR.pack(g.random(S.N_VOXELS) < d) for d in (0.0, 0.1, 0.3, 1.0, 0.5)]
    for with_inv in (False, True):
        got = S.completion_counts(np.stack(preds), np.stack(labs), np.stack(invs) if with_inv else None)
        want = [SR.confusion(p, l, i if with_inv else None) for p, l, i in zip(preds, labs, invs)]
        assert got.tolist() == [list(w) for w in want]
        for p, l, i, w in zip(preds, labs, invs, want):
            assert tuple(S.completion_counts(p, l, i if with_inv else None)) == w
    full = np.full(S.N_VOXELS, 1, np.uint16)
    assert tuple(S.completion_counts(SR.pack(np.ones(S.N_VOXELS, bool)), full)) == (S.N_VOXELS, 0, 0)


def test_eval_path_voxels_and_ssc_end_to_end(tmp_path):
    from click.testing import CliRunner
    from ssc_sequence import SCORED, make_voxel_sequence
    from lidiff_b200.synth import read_ply_xyz
    from lidiff_b200.tools.eval_path import main
    seq, grids, sub, plys = make_voxel_sequence(tmp_path)
    logs = {}
    for name, args in (("voxels", ["-p", grids + "/", "--data", seq, "--voxels"]), ("plys", ["-p", plys + "/", "--data", sub]),
                       ("ssc", ["-p", grids + "/", "--data", seq, "--voxels", "--ssc"]),
                       ("points_ssc", ["-p", os.path.join(str(tmp_path), "pred") + "/", "--data", seq, "--ssc"])):
        res = CliRunner().invoke(main, args, catch_exceptions=False)
        assert res.exit_code == 0, res.output
        log = os.path.join(args[1], "res_log.yaml")
        logs[name] = json.load(open(log))
        os.remove(log)
    assert logs["voxels"] == logs["plys"] and np.isfinite(logs["voxels"]["cd_mean"]) and "ssc_iou" not in logs["voxels"]
    ssc = logs["ssc"]
    assert {k: v for k, v in ssc.items() if not k.startswith("ssc_")} == logs["voxels"]
    tp = fp = fn = 0
    for j, b in enumerate(SCORED):
        stem = os.path.join(seq, "voxels", f"{b:06d}")
        occ = SR.unpack(SR.voxelize(read_ply_xyz(os.path.join(plys, f"{j:06d}.ply")))[0])
        c = SR.confusion(SR.pack(occ), np.fromfile(stem + ".label", "<u2"), np.fromfile(stem + ".invalid", "<u4"))
        tp, fp, fn = tp + c[0], fp + c[1], fn + c[2]
    assert ssc["ssc_iou"] == tp / (tp + fp + fn) and ssc["ssc_precision"] == tp / (tp + fp + 1e-8)
    assert ssc["ssc_recall"] == tp / (tp + fn + 1e-8) and 0 < ssc["ssc_iou"] < 1
    assert 0 < logs["points_ssc"]["ssc_iou"] < 1 and "cd_mean" in logs["points_ssc"]


def test_kernels_run_on_the_device():
    h = _lib.get_handle("cuda")
    l0 = h.launch_count()
    lab = np.zeros(S.N_VOXELS, np.uint16)
    lab[5] = 1
    pts, _ = S.grid_points(lab, "labels")
    bits, _ = S.voxelize(pts)
    S.completion_counts(bits, lab)
    assert h.launch_count() - l0 == 4 + 1 + 1
