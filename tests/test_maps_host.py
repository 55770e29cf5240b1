"""Host logic of lidiff_b200.maps and the map_from_scans CLI on the numpy stand-in backend (tests/fake_maps_backend.py): options,
file naming, the reference's pose / scan pairing (truncation, missing calib.txt), missing labels, growth, rank splits, and the
streaming build against a one-shot global first-occurrence de-duplication and against the reference's recorded maps."""
import os
import shutil
import socket
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp
from click.testing import CliRunner

import fake_maps_backend
from fake_maps_backend import restate_map
from lidiff_b200 import kitti
from lidiff_b200.maps import MapBuilder
from lidiff_b200.tools import map_from_scans as MS

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_map_goldens as G  # noqa: E402


@pytest.fixture
def fake(monkeypatch):
    return fake_maps_backend.install(monkeypatch)


def _pose12(p):
    return p[:3, :4].astype(np.float32).reshape(-1)


def _expected(seq_dir, div_mode=1, voxel=0.1):
    """the restated map of a sequence: scans paired with poses as the reference pairs them"""
    poses = kitti.load_poses(os.path.join(seq_dir, "calib.txt"), os.path.join(seq_dir, "poses.txt"))
    names = kitti.natural_sorted(os.listdir(os.path.join(seq_dir, "velodyne")))
    scans = []
    for pose, name in zip(poses, names):
        path = os.path.join(seq_dir, "velodyne", name)
        scans.append((kitti.read_scan(path), kitti.read_labels(kitti.label_path(path)), _pose12(pose)))
    return restate_map(scans, voxel, div_mode)


def _run(args):
    return CliRunner().invoke(MS.main, args)


def test_cli_options_and_no_cpu_path():
    out = _run(["--help"]).output
    for opt in ("--path", "-p", "--voxel_size", "-v", "--cpu", "-c", "--sequences", "--div-mode"):
        assert opt in out
    res = _run(["-p", "x", "-c"])
    assert res.exit_code == 2 and "no CPU path" in res.output


def test_cli_writes_each_sequence_map(fake, tmp_path):
    for i, seq in enumerate(["00", "01", "02"]):
        G.write_sequence(str(tmp_path / seq), seed=i)
    res = _run(["-p", str(tmp_path), "--sequences", "00,02", "-v", "0.2", "--div-mode", "0"])
    assert res.exit_code == 0, res.output
    assert res.output.splitlines() == ["saving map for sequence 00", "saving map for sequence 02"]
    assert not (tmp_path / "01" / "map_clean.npy").exists()
    for seq in ("00", "02"):
        m = np.load(tmp_path / seq / "map_clean.npy")
        assert m.dtype == np.float32 and m.ndim == 2 and m.shape[1] == 3 and m.shape[0] > 1000
        assert np.array_equal(m, _expected(str(tmp_path / seq), div_mode=0, voxel=0.2))


def test_default_sequences_are_00_to_10():
    assert MS.parse_sequences(()) == G.SEQUENCES
    assert MS.parse_sequences(("00", "03,08")) == ["00", "03", "08"]


@pytest.mark.parametrize("n_scans,n_poses", [(3, 5), (4, 2)])
def test_scans_and_poses_are_zipped_to_the_shorter(fake, tmp_path, n_scans, n_poses):
    seq = str(tmp_path / "00")
    G.write_sequence(seq, n_scans=n_scans, n_poses=n_poses)
    assert len(MS.sequence_scans(seq)) == min(n_scans, n_poses)
    got = MS.build_sequence_map(seq, device="cpu")
    assert np.array_equal(got, _expected(seq))
    full = MapBuilder(device="cpu")
    for pose, path in MS.sequence_scans(seq)[: min(n_scans, n_poses) - 1]:
        full.add_scan(kitti.read_scan(path), kitti.read_labels(kitti.label_path(path)), pose)
    assert full.n < got.shape[0]                                  # the last paired scan contributes


def test_missing_calib_leaves_poses_untransformed(fake, tmp_path):
    seq = str(tmp_path / "03")
    G.write_sequence(seq, calib=False)
    raw = np.loadtxt(os.path.join(seq, "poses.txt")).reshape(-1, 3, 4)
    for (pose, _), p in zip(MS.sequence_scans(seq), raw):
        assert np.array_equal(pose[:3], p)
    assert np.array_equal(MS.build_sequence_map(seq, device="cpu"), _expected(seq))


def test_missing_label_file_is_named(fake, tmp_path):
    seq = tmp_path / "00"
    G.write_sequence(str(seq))
    os.remove(seq / "labels" / "000001.label")
    res = _run(["-p", str(tmp_path), "--sequences", "00"])
    assert res.exit_code != 0
    assert isinstance(res.exception, FileNotFoundError) and "000001.label" in str(res.exception)


def test_streaming_equals_one_shot_and_growth(fake, tmp_path):
    seq = str(tmp_path / "00")
    G.write_sequence(seq, n_scans=5, margin=0)
    scans = [(kitti.read_scan(p), kitti.read_labels(kitti.label_path(p)), pose) for pose, p in MS.sequence_scans(seq)]
    small, big = MapBuilder(device="cpu", initial_capacity=1), MapBuilder(device="cpu", initial_capacity=1 << 16)
    for pts, lab, pose in scans:
        small.add_scan(pts, lab, pose)
        big.add_scan(pts, lab, pose)
    assert small.rehashes >= 3 and big.rehashes == 0
    assert np.array_equal(small.points().numpy(), big.points().numpy())
    assert np.array_equal(small.points().numpy(), restate_map([(p, l, _pose12(q)) for p, l, q in scans], 0.1, 1))


def test_out_of_range_key_raises_and_poisons_the_builder(fake):
    mb = MapBuilder(device="cpu")
    far = np.array([[4.0, 0, 0, 0], [2.0 ** 20 * 0.1 + 1.0, 0, 0, 0]], np.float32)
    with pytest.raises(ValueError, match="key range"):
        mb.add_scan(far)
    with pytest.raises(RuntimeError):
        mb.add_scan(far[:1])


def test_fake_cli_reproduces_the_reference_golden(fake, tmp_path):
    ref = np.load(os.path.join(HERE, "golden", "map_reference.npz"))
    G.make_dataset(str(tmp_path), int(ref["seed"]))
    res = _run(["-p", str(tmp_path), "--div-mode", "0", "-v", str(float(ref["voxel_size"]))])
    assert res.exit_code == 0, res.output
    for seq in G.SEQUENCES:
        got, want = np.load(tmp_path / seq / "map_clean.npy"), ref[f"seq{seq}"]
        assert got.shape == want.shape, seq
        assert np.abs(got - want).max() <= 1e-5, seq


def _worker(rank, world, port, root, q):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": "0"})
    from lidiff_b200 import _lib
    h = fake_maps_backend.FakeMapsHandle()
    _lib.get_handle = lambda device=None: h
    MS.main(["-p", root, "--sequences", "00,01,02,03"], standalone_mode=False)
    q.put(rank)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def test_maps_do_not_depend_on_the_world_size(tmp_path):
    src = tmp_path / "src"
    for i, seq in enumerate(["00", "01", "02", "03"]):
        G.write_sequence(str(src / seq), n_scans=2, seed=10 + i, azimuths=64)
    maps = {}
    ctx = mp.get_context("spawn")
    for world in (1, 2, 3):
        root = str(tmp_path / f"w{world}")
        shutil.copytree(src, root)
        q = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, world, port, root, q)) for r in range(world)]
        for p in procs:
            p.start()
        done = sorted(q.get(timeout=180) for _ in range(world))
        for p in procs:
            p.join(timeout=60)
        assert done == list(range(world)) and all(p.exitcode == 0 for p in procs)
        maps[world] = {seq: np.load(os.path.join(root, seq, "map_clean.npy")) for seq in ("00", "01", "02", "03")}
    for world in (2, 3):
        for seq in maps[1]:
            assert np.array_equal(maps[world][seq], maps[1][seq]), (world, seq)
