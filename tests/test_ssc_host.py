"""Host tests of the SemanticKITTI scene-completion grids (lidiff_b200.ssc) and `eval_path --voxels / --ssc` on the CPU stand-in
backend: file sizes, the MSB-first bit order of a hand-written `.bin`, the label rules, invalid masking, point -> voxel at the
extent's edges, round trips, and the CLI's results against scoring `.ply` files of the same voxel centres."""
import os

import numpy as np
import pytest
import torch

import fake_ssc_backend
import ssc_reference as SR
from lidiff_b200 import metrics as M
from lidiff_b200 import ssc as S
from lidiff_b200.tools import eval_path as E


@pytest.fixture
def fake(monkeypatch):
    return fake_ssc_backend.install(monkeypatch)


def _v(i, j, k):
    return (i * 256 + j) * 32 + k


def test_constants_match_the_header_and_the_reference():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "lidiff_b200.h")).read()
    for name, val in (("DIM_X", "256"), ("DIM_Y", "256"), ("DIM_Z", "32"), ("VOXELS", "2097152"), ("WORDS", "65536"),
                      ("VOXEL", "0.2"), ("MIN_X", "0.0"), ("MIN_Y", "(-25.6)"), ("MIN_Z", "(-2.0)"), ("IGNORE", "255")):
        assert hdr.split(f"#define LB2_SSC_{name} ")[1].split()[0] == val, name
    assert S.DIMS == SR.DIMS and S.N_VOXELS == SR.N_VOXELS == np.prod(S.DIMS) and S.N_WORDS * 32 == S.N_VOXELS
    assert S.BIN_BYTES == 262144 and S.LABEL_BYTES == 4194304
    assert np.array_equal(np.array(S.GRID_MIN) + np.array(S.DIMS) * S.VOXEL_SIZE, S.GRID_MAX)


# ---- files --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,size", [("a.label", 4194303), ("a.label", 262144), ("a.bin", 262145), ("a.invalid", 4194304),
                                       ("a.bin", 0)])
def test_wrong_size_raises_naming_the_file_and_its_size(tmp_path, name, size):
    p = tmp_path / name
    p.write_bytes(b"\0" * size)
    with pytest.raises(ValueError, match=rf"{name}: {size} bytes"):
        S.read_grid(str(p))


def test_read_and_write_round_trip(tmp_path):
    g = np.random.default_rng(0)
    words = g.integers(0, 2 ** 32, S.N_WORDS, dtype=np.uint64).astype(np.uint32)
    S.write_bin(str(tmp_path / "a.bin"), words)
    S.write_bin(str(tmp_path / "b.invalid"), torch.from_numpy(words.view(np.int32)))
    assert (tmp_path / "a.bin").read_bytes() == words.tobytes() == (tmp_path / "b.invalid").read_bytes()
    got, kind = S.read_grid(str(tmp_path / "a.bin"))
    assert kind == "bits" and np.array_equal(got, words) and np.array_equal(S.read_invalid(str(tmp_path / "b.invalid")), words)
    lab = g.integers(0, 2 ** 16, S.N_VOXELS, dtype=np.uint16)
    lab.astype("<u2").tofile(str(tmp_path / "a.label"))
    got, kind = S.read_grid(str(tmp_path / "a.label"))
    assert kind == "labels" and np.array_equal(got, lab)
    with pytest.raises(ValueError, match="a grid has 262144"):
        S.write_bin(str(tmp_path / "c.bin"), words[:-1])
    with pytest.raises(ValueError, match="a .label, .bin or .invalid"):
        S.read_grid(str(tmp_path / "a.ply"))


def test_hand_written_bin_bit_order(fake, tmp_path):
    """bit 7 - (v & 7) of byte v >> 3: 0x80 in byte 0 is voxel 0, 0x01 voxel 7, 0x40 in byte 1 voxel 9, 0x01 in the last byte
    the last voxel"""
    raw = bytearray(S.BIN_BYTES)
    raw[0] = 0x81
    raw[1] = 0x40
    raw[_v(3, 200, 16) >> 3] = 0x80                                   # k = 16: the first voxel of a byte
    raw[-1] = 0x01
    (tmp_path / "h.bin").write_bytes(bytes(raw))
    bits, kind = S.read_grid(str(tmp_path / "h.bin"))
    pts, off = S.grid_points(bits, kind, device="cpu")
    want_v = [0, 7, 9, _v(3, 200, 16), S.N_VOXELS - 1]
    assert list(off) == [0, 5]
    i, j, k = np.array(want_v) // 8192, (np.array(want_v) // 32) % 256, np.array(want_v) % 32
    want = np.stack([0.0 + (i + 0.5) * 0.2, -25.6 + (j + 0.5) * 0.2, -2.0 + (k + 0.5) * 0.2], 1)
    assert np.array_equal(pts.numpy(), want)
    assert np.array_equal(pts.numpy()[0], [0.1, -25.5, -1.9]) and np.allclose(pts.numpy()[-1], [51.1, 25.5, 4.3], atol=1e-12)
    assert np.array_equal(np.flatnonzero(SR.unpack(bits)), want_v)
    vox = S.voxelize(pts, device="cpu")[0].numpy().view(np.uint32)
    assert vox.tobytes() == bytes(raw)                                # the device words are the file's little-endian bytes


def test_label_rules(fake):
    lab = np.zeros(S.N_VOXELS, np.uint16)
    vals = {3: 255, 4: 1, 5: 254, 6: 256, 7: 65535, 8: 0, 40: 40}
    for v, x in vals.items():
        lab[v] = x
    pts, off = S.grid_points(lab, "labels", device="cpu")
    assert list(off) == [0, 5] and np.array_equal(pts.numpy(), SR.centres(np.isin(np.arange(S.N_VOXELS), [4, 5, 6, 7, 40])))


def test_several_grids_and_chunks(fake, monkeypatch):
    monkeypatch.setattr(S, "CHUNK", 2)
    g = np.random.default_rng(1)
    grids = [SR.random_labels(g, d) for d in (0.0, 1e-4, 0.01, 0.0)] + [np.full(S.N_VOXELS, 7, np.uint16)]
    l0 = fake.launches
    pts, off = S.grid_points(grids, "labels", device="cpu")
    assert fake.launches - l0 == 3 * 4                               # 3 chunks: three counting launches and one emit each
    want = [SR.centres(SR.occupied(x)) for x in grids]
    assert list(np.diff(off)) == [w.shape[0] for w in want] and off[-1] == sum(w.shape[0] for w in want)
    assert np.array_equal(pts.numpy(), np.concatenate(want))
    with pytest.raises(ValueError, match="labels grids"):
        S.grid_points(np.zeros(10, np.uint16), "labels", device="cpu")
    with pytest.raises(ValueError, match="kind"):
        S.grid_points(grids[0], "points", device="cpu")


# ---- point -> voxel -----------------------------------------------------------------------------------------------------------
def test_point_to_voxel_at_the_extent_edges(fake):
    nan, inf = float("nan"), float("inf")
    rows = np.array([[0.0, 0.0, 0.0], [-0.0, -0.0, -0.0], [51.2, 0.0, 0.0], [np.nextafter(51.2, 0), 0.0, 0.0],
                     [1.0, -25.6, 0.0], [1.0, 25.6, 0.0], [1.0, 0.0, -2.0], [1.0, 0.0, 4.4], [1.0, 0.0, np.nextafter(4.4, 0)],
                     [-1e-300, 0.0, 0.0], [nan, 0.0, 0.0], [0.0, inf, 0.0], [0.0, 0.0, -inf], [1e300, 0.0, 0.0], [0.2, 0.0, 0.0]])
    v, nf, out = SR.voxel_index(rows)
    kept = {0: _v(0, 128, 10), 1: _v(0, 128, 10), 3: _v(255, 128, 10), 4: _v(5, 0, 10), 6: _v(5, 128, 0), 8: _v(5, 128, 31),
            14: _v(1, 128, 10)}
    assert {i: int(x) for i, x in enumerate(v) if x >= 0} == kept
    assert list(np.flatnonzero(nf)) == [10, 11, 12] and list(np.flatnonzero(out)) == [2, 5, 7, 9, 13]
    bits, dropped = S.voxelize(rows, device="cpu")
    assert list(dropped) == [3, 5]
    assert np.array_equal(np.flatnonzero(SR.unpack(bits.numpy().view(np.uint32))), sorted(set(kept.values())))


def test_round_trips(fake):
    g = np.random.default_rng(2)
    for lab in (SR.random_labels(g, 0.03, 0.01), np.full(S.N_VOXELS, 9, np.uint16)):
        pts, _ = S.grid_points(lab, "labels", device="cpu")
        bits, dropped = S.voxelize(pts, device="cpu")
        assert np.array_equal(bits.numpy().view(np.uint32), SR.pack(SR.occupied(lab))) and list(dropped) == [0, 0]
        again, _ = S.grid_points(bits, "bits", device="cpu")
        assert np.array_equal(again.numpy(), pts.numpy())
    cloud = np.concatenate([g.uniform([-5, -30, -3], [55, 30, 5], (50000, 3)), [[np.nan, 1, 1]]])
    v, _, _ = SR.voxel_index(cloud)
    bits, dropped = S.voxelize(cloud, device="cpu")
    centres = S.grid_points(bits, "bits", device="cpu")[0].numpy()
    assert dropped[0] == 1 and dropped[1] == int((v < 0).sum()) - 1
    kept = cloud[v >= 0]
    own = SR.GRID_MIN + (np.floor((kept - SR.GRID_MIN) / 0.2) + 0.5) * 0.2   # each kept point's voxel centre
    assert np.array_equal(np.unique(own, axis=0), np.unique(centres, axis=0)) and centres.shape[0] == np.unique(v[v >= 0]).shape[0]


def test_voxelize_batches_and_offsets(fake):
    g = np.random.default_rng(3)
    clouds = [g.uniform(0, 20, (n, 3)) for n in (5, 0, 300)]
    off = np.cumsum([0] + [c.shape[0] for c in clouds])
    bits, dropped = S.voxelize(np.concatenate(clouds), off, device="cpu")
    assert bits.shape == (3, S.N_WORDS) and dropped.shape == (3, 2)
    for c, b in zip(clouds, bits):
        assert np.array_equal(b.numpy().view(np.uint32), SR.voxelize(c)[0])
    for bad in ([0, 5], [1, 305], [0, 10, 5, 305]):
        with pytest.raises(ValueError, match="offsets"):
            S.voxelize(np.concatenate(clouds), bad, device="cpu")


# ---- completion counts ----------------------------------------------------------------------------------------------------------
def test_completion_counts_hand_counted(fake):
    lab = np.zeros(S.N_VOXELS, np.uint16)
    lab[[10, 11, 12, 13]] = [40, 40, 40, 40]                          # 13 is occupied but invalid
    lab[20] = 255
    inv = np.zeros(S.N_VOXELS, bool)
    inv[[13, 30]] = True
    pred = np.zeros(S.N_VOXELS, bool)
    pred[[10, 11, 13, 20, 30, 31]] = True                             # TP 10, 11; FP 31 (20 ignored, 13 and 30 invalid); FN 12
    assert list(S.completion_counts(SR.pack(pred), lab, SR.pack(inv), device="cpu")) == [2, 1, 1]
    assert list(S.completion_counts(SR.pack(pred), lab, device="cpu")) == [3, 2, 1]    # without the mask: 13 TP, 30 FP
    stacked = S.completion_counts(np.stack([SR.pack(pred)] * 2), np.stack([lab, lab]), np.stack([SR.pack(inv)] * 2), device="cpu")
    assert stacked.tolist() == [[2, 1, 1], [2, 1, 1]]
    acc = S.SSCCompletion()
    acc.add([2, 1, 1])
    acc.add([3, 2, 1])
    r = acc.compute()
    assert acc.scans == 2 and r["iou"] == 5 / 10 and r["precision"] == 5 / (8 + 1e-8) and r["recall"] == 5 / (7 + 1e-8)
    assert np.isnan(S.SSCCompletion().compute()["iou"])


# ---- eval_path --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def voxel_sequence(tmp_path_factory):
    from ssc_sequence import make_voxel_sequence
    return make_voxel_sequence(tmp_path_factory.mktemp("ssc"))


def _res(local, ssc=False):
    return E.to_json(E.fold({k: M.record_from_rows(r[:-3] if ssc else r) for k, r in local.items()}, verbose=False))


def test_eval_path_voxels_equals_scoring_the_voxel_centres(fake, voxel_sequence):
    seq, grids, sub, plys = voxel_sequence
    l0 = fake.launches
    n, a = E.score_scans(seq, grids + "/", None, 50.0, "refine", "cpu", voxels=True)
    assert n == 3 and sorted(a) == [0, 1, 2]
    n2, b = E.score_scans(sub, plys + "/", None, 50.0, "refine", "cpu")
    assert n2 == 3 and _res(a) == _res(b) and np.isfinite(_res(a)["cd_mean"])
    assert all(torch.equal(a[k], b[k]) for k in a)
    split = {}
    for rank in range(3):                                             # the rank split does not change the records
        split.update(E.score_scans(seq, grids, None, 50.0, "refine", "cpu", rank=rank, world=3, voxels=True)[1])
    assert sorted(split) == [0, 1, 2] and all(torch.equal(split[k], a[k]) for k in a)
    assert fake.launches > l0


def test_eval_path_ssc_counts(fake, voxel_sequence):
    from lidiff_b200.synth import read_ply_xyz
    seq, grids, sub, plys = voxel_sequence
    _, a = E.score_scans(seq, grids, None, 50.0, "refine", "cpu", voxels=True, ssc=True)
    _, plain = E.score_scans(seq, grids, None, 50.0, "refine", "cpu", voxels=True)
    assert _res(a, ssc=True) == _res(plain)                           # the SSC rows leave the other metrics alone
    counts = {k: E.ssc_from_rows(r[-3:]) for k, r in a.items()}
    for j, b in enumerate((0, 5, 10)):
        stem = os.path.join(seq, "voxels", f"{b:06d}")
        occ = SR.unpack(SR.voxelize(read_ply_xyz(os.path.join(plys, f"{j:06d}.ply")))[0])
        want = SR.confusion(SR.pack(occ), np.fromfile(stem + ".label", "<u2"), np.fromfile(stem + ".invalid", "<u4"))
        assert list(counts[j]) == [1, *want]
    res = E.fold_ssc(counts)
    tp, fp, fn = (sum(int(c[i]) for c in counts.values()) for i in (1, 2, 3))
    assert res == {"ssc_iou": tp / (tp + fp + fn), "ssc_precision": tp / (tp + fp + 1e-8), "ssc_recall": tp / (tp + fn + 1e-8)}
    # point predictions of every scan: only the scans with a ground-truth grid count
    seq_pred = os.path.join(os.path.dirname(seq), "pred")
    n, p = E.score_scans(seq, seq_pred, None, 50.0, "refine", "cpu", ssc=True)
    assert n == 11 and [int(E.ssc_from_rows(p[b][-3:])[0]) for b in range(11)] == [int(b % 5 == 0) for b in range(11)]


def test_eval_path_ssc_hand_counted(fake, tmp_path):
    """one scan: ground truth occupied at voxels a, b, c, 255 at d, invalid at e (occupied); the prediction has points in a, b,
    d, e and f, one outside the grid and one NaN: TP 2, FP 1 (f), FN 1 (c)"""
    a, b, c, d, e, f = (_v(10, 128, 10), _v(10, 128, 11), _v(20, 100, 5), _v(30, 30, 3), _v(40, 200, 20), _v(50, 7, 8))
    (tmp_path / "voxels").mkdir()
    lab = np.zeros(S.N_VOXELS, "<u2")
    lab[[a, b, c, e]] = 40
    lab[d] = 255
    lab.tofile(str(tmp_path / "voxels" / "000000.label"))
    inv = np.zeros(S.N_VOXELS, bool)
    inv[e] = True
    SR.pack(inv).tofile(str(tmp_path / "voxels" / "000000.invalid"))
    pred = np.concatenate([SR.centres(np.isin(np.arange(S.N_VOXELS), [a, b, d, e, f])), [[60.0, 0, 0], [np.nan, 0, 0]]])
    assert list(E.ssc_counts(str(tmp_path), "000000.bin", pred, "cpu")) == [1, 2, 1, 1]
    assert list(E.ssc_counts(str(tmp_path), "000001.bin", pred, "cpu")) == [0, 0, 0, 0]
    rows = E.ssc_to_rows(np.array([1, 2, 1, 1]))
    assert rows.shape == (3, 3) and rows.dtype == torch.float32 and list(E.ssc_from_rows(rows)) == [1, 2, 1, 1]
    assert E.fold_ssc({0: np.array([1, 2, 1, 1]), 1: np.array([0, 0, 0, 0])}) == \
        {"ssc_iou": 0.5, "ssc_precision": 2 / (3 + 1e-8), "ssc_recall": 2 / (3 + 1e-8)}


def test_eval_path_voxels_needs_grids_and_ssc_needs_ground_truth(fake, voxel_sequence, tmp_path):
    seq, grids, sub, plys = voxel_sequence
    empty = tmp_path / "empty"
    empty.mkdir()
    with pytest.raises(FileNotFoundError, match="no <stem>.label or <stem>.bin grid"):
        E.score_scans(seq, str(empty), None, 50.0, "refine", "cpu", voxels=True)
    with pytest.raises(FileNotFoundError, match="--ssc: no ground-truth grid"):
        E.score_scans(sub, plys, None, 50.0, "refine", "cpu", ssc=True)


def test_eval_path_voxels_options():
    from click.testing import CliRunner
    for extra in (["--mesh"], ["--random-weights"], ["-d", "x.ckpt"], ["-r", "y.ckpt"]):
        res = CliRunner().invoke(E.main, ["-p", "x/", "--voxels", *extra])
        assert res.exit_code != 0 and "--voxels scores grid files" in res.output
    res = CliRunner().invoke(E.main, ["--help"])
    assert "--voxels" in res.output and "--ssc" in res.output


def test_completion_pipeline_has_the_ssc_option():
    from click.testing import CliRunner
    from lidiff_b200.tools.diff_completion_pipeline import main
    assert "--ssc" in CliRunner().invoke(main, ["--help"]).output
