"""Records the ground-truth maps the reference's `lidiff/map_from_scans.py` builds on a seeded synthetic 11-sequence dataset, so
lidiff_b200.maps / tools.map_from_scans can be compared against them without the reference's source tree:

    python tests/golden/make_map_goldens.py REF        # REF = a checkout of the reference -> tests/golden/map_reference.npz

The reference's script runs unchanged (`-p DATA -c`: the CPU, i.e. true division by the voxel size) on the shims.  One stand-in:
`ME.utils.sparse_quantize` is replaced by a first-occurrence de-duplication that floors the coordinates, as MinkowskiEngine does
for float coordinates (`_auto_floor`); the shim's version truncates toward zero, which merges the voxels on either side of 0 and so
would record a different map.  The dataset is regenerated from the seed by `make_dataset()`; only the maps are stored.

Every transformed point is kept at least MARGIN = 1e-4 m (checked in fp64) from a voxel face and from the 3.5 m range boundary, so
the order in which the host BLAS sums the pose product cannot change which voxel a point falls in or whether it is kept.  The data
covers: negative coordinates, duplicates within a scan and across scans, remission that decides the range filter, every excluded
label class with instance ids in the upper bits, a sequence without calib.txt, one with more poses than scans and one with more scans
than poses.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

SEED = 7
VOXEL = 0.1
MARGIN = 1e-4
SEQUENCES = ["00", "01", "02", "03", "04", "05", "06", "07", "08", "09", "10"]
TR = np.array([[0.0, -1.0, 0.0, 0.1], [0.0, 0.0, -1.0, -0.05], [1.0, 0.0, 0.0, -0.3], [0.0, 0.0, 0.0, 1.0]])   # LiDAR -> camera
EXCLUDED = [0, 1, 252, 253, 254, 255, 256, 257, 258, 259, 0xFFFF]
KEPT = [2, 9, 10, 11, 40, 44, 48, 50, 51, 70, 71, 72, 80, 81, 99, 251]


def lidar_pose(b, turn=0.07, step=(1.5, 0.4, 0.05)):
    a = turn * b
    return np.array([[np.cos(a), -np.sin(a), 0.0, step[0] * b], [np.sin(a), np.cos(a), 0.0, step[1] * b], [0, 0, 1.0, step[2] * b],
                     [0, 0, 0, 1.0]])


def _transform64(pose32, pts):
    return pts[:, :3].astype(np.float64) @ pose32[:3, :3].T.astype(np.float64) + pose32[:3, 3].astype(np.float64)


def _clear_of_faces(pose32, pts, voxel, margin):
    """fp64: every transformed coordinate at least `margin` from a voxel face, and |(x, y, z, r)| at least `margin` from 3.5"""
    w = _transform64(pose32, pts)
    q = w / voxel
    face = np.abs(q - np.round(q)).min(1) * voxel >= margin
    rng = np.abs(np.sqrt((pts.astype(np.float64) ** 2).sum(1)) - 3.5) >= margin
    return face & rng


def write_sequence(seq_dir, n_scans=3, n_poses=None, calib=True, seed=0, beams=16, azimuths=96, voxel=VOXEL, margin=MARGIN,
                   labels=True):
    """a KITTI-layout sequence: velodyne/*.bin, labels/*.label, poses.txt (camera frame through Tr when calib.txt is written) and
    calib.txt; returns the LiDAR-frame poses as the readers see them"""
    from lidiff_b200.kitti import load_poses
    from lidiff_b200.synth import synthetic_scan
    n_poses = n_scans if n_poses is None else n_poses
    os.makedirs(os.path.join(seq_dir, "velodyne"), exist_ok=True)
    if labels:
        os.makedirs(os.path.join(seq_dir, "labels"), exist_ok=True)
    g = np.random.default_rng(seed)
    if calib:
        with open(os.path.join(seq_dir, "calib.txt"), "w") as f:
            f.write("P0: " + " ".join(["0"] * 12) + "\n")
            f.write("Tr: " + " ".join(f"{v:.12e}" for v in TR[:3].reshape(-1)) + "\n")
    with open(os.path.join(seq_dir, "poses.txt"), "w") as f:
        for b in range(n_poses):
            p = lidar_pose(b)
            cam = TR @ p @ np.linalg.inv(TR) if calib else p
            f.write(" ".join(f"{v:.12e}" for v in cam[:3].reshape(-1)) + "\n")
    poses = load_poses(os.path.join(seq_dir, "calib.txt"), os.path.join(seq_dir, "poses.txt"))
    prev_world = None
    for b in range(n_scans):
        pose = poses[min(b, len(poses) - 1)]
        xyz = synthetic_scan(seed * 100 + b, beams=beams, azimuths=azimuths)
        n = xyz.shape[0]
        r = g.uniform(0, 1, (n, 1))
        near = g.normal(size=(64, 3))                                        # around the 3.5 m boundary; remission decides some
        near = near / np.linalg.norm(near, axis=1, keepdims=True) * g.uniform(2.5, 4.0, (64, 1))
        rows = [np.concatenate([xyz, r], 1), np.concatenate([near, g.uniform(0, 2.5, (64, 1))], 1)]
        if prev_world is not None:                                           # points of the previous scan seen again: same world voxel
            back = (prev_world[: n // 4] - pose[:3, 3]) @ pose[:3, :3]
            rows.append(np.concatenate([back, g.uniform(0, 1, (back.shape[0], 1))], 1))
        pts = np.concatenate(rows)
        pts = np.concatenate([pts, pts[g.choice(pts.shape[0], pts.shape[0] // 10)],          # exact duplicates within the scan
                              pts[g.choice(pts.shape[0], pts.shape[0] // 10)] + g.uniform(-0.01, 0.01, (pts.shape[0] // 10, 4))])
        pts = pts[g.permutation(pts.shape[0])].astype(np.float32)
        if margin:
            pts = pts[_clear_of_faces(pose.astype(np.float32), pts, voxel, margin)]
        cls = np.where(g.uniform(size=pts.shape[0]) < 0.25, g.choice(EXCLUDED, pts.shape[0]), g.choice(KEPT, pts.shape[0]))
        lab = (cls.astype(np.uint32) | (g.integers(0, 1 << 16, pts.shape[0]).astype(np.uint32) << 16)).astype(np.uint32)
        pts.tofile(os.path.join(seq_dir, "velodyne", f"{b:06d}.bin"))
        if labels:
            lab.tofile(os.path.join(seq_dir, "labels", f"{b:06d}.label"))
        prev_world = _transform64(pose.astype(np.float32), pts)[(lab & 0xFFFF) > 1]
    return poses


def make_dataset(root, seed=SEED):
    """11 sequences 00..10 under root: 03 has no calib.txt, 04 one pose more than scans, 05 one scan more than poses"""
    for i, seq in enumerate(SEQUENCES):
        write_sequence(os.path.join(root, seq), n_scans=3 + (i == 5), n_poses=3 + (i == 4), calib=i != 3, seed=seed * 1000 + i)
    return root


def flooring_sparse_quantize(coordinates, features=None, return_index=False, quantization_size=None, **_):
    """ME.utils.sparse_quantize on float coordinates: floor, then the first occurrence of every voxel (indices ascending)"""
    import torch
    c = torch.floor(torch.as_tensor(coordinates) if quantization_size is None else torch.as_tensor(coordinates) / quantization_size)
    c = c.to(torch.int64)
    _, inv = torch.unique(c, dim=0, return_inverse=True)
    first = torch.full((int(inv.max()) + 1 if inv.numel() else 0,), c.shape[0], dtype=torch.long)
    first.scatter_reduce_(0, inv, torch.arange(c.shape[0]), "amin")
    first = torch.sort(first).values
    return (c[first].int(), first) if return_index else c[first].int()


def main(ref):
    import importlib
    import lidiff_b200.shims as sh
    sh.install()
    import MinkowskiEngine as ME
    ME.utils.sparse_quantize = flooring_sparse_quantize
    sys.path.insert(0, ref)
    for k in [k for k in sys.modules if k == "lidiff" or k.startswith("lidiff.")]:
        sys.modules.pop(k)
    script = importlib.import_module("lidiff.map_from_scans")
    with tempfile.TemporaryDirectory() as root:
        make_dataset(root)
        script.main(["-p", root, "-c"], standalone_mode=False)
        maps = {f"seq{seq}": np.load(os.path.join(root, seq, "map_clean.npy")) for seq in SEQUENCES}
    np.savez_compressed(os.path.join(HERE, "map_reference.npz"), seed=np.array(SEED), voxel_size=np.array(VOXEL), **maps)
    print({k: v.shape for k, v in maps.items()})


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
