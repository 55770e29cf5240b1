"""Records the samples the reference's `TemporalKITTISet` (lidiff/datasets/dataloader/SemanticKITTITemporal.py) builds on a seeded
synthetic SemanticKITTI layout, so lidiff_b200.datasets can be compared against them without the reference's source tree:

    python tests/golden/make_sample_goldens.py REF        # REF = a checkout of the reference -> tests/golden/samples_reference.npz

The reference's class runs unchanged on the shims, with three stand-ins: `hdbscan` and `matplotlib` (imported by
utils/pcd_preprocess.py, never called here) are empty modules, and the open3d shim's farthest_point_down_sample (GPU only) is the
oracle's numpy farthest point sampling (oracle/pipeline.py, the same open3d semantics).  The dataset is regenerated from the seed by
`make_dataset()`; only the samples are stored.

Every scan point is kept at least GEN_MARGIN from the 3.5 m / max_range boundaries and from z = -4, and every map point as far from
the crop radius and from z = -4 in the frame of every pose, so the order in which a BLAS sums the pose product cannot change a
decision.  The viewpoint grid's cells depend on the augmentation, so they are checked rather than generated: the recording fails
if a grid point or a query lies within CELL_MARGIN of a 10 m cell face (larger than a float32 ulp at the coordinates used, so an
augmentation that rounds differently by one ulp cannot move a point across a face either); the recorded decisions of the range
and height filters are asserted to be at least CHECK_MARGIN from their boundaries.  Covered: excluded label classes with instance
bits, NaN / inf rows, points below z = -4 and beyond max_range, a partial scan shorter than num_points / 10 (element-wise repeat), a
viewpoint-filtered map both shorter and longer than num_points (repeat / truncation), and the train, validation and test splits.
"""
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SEED = 11
NUM_POINTS = 4000
MAX_RANGE = 50.0
RESOLUTION = 0.05
GEN_MARGIN = 1e-4
CHECK_MARGIN = 1e-6
CELL_MARGIN = 1e-5
SEQUENCES = {"00": 3, "01": 2, "08": 3}                      # name -> scans
TRAIN, VALIDATION = ["00", "01"], ["08"]
RECORD = {"train": [0, 4], "validation": [1, 0], "test": [1, 2]}   # indices recorded per split, in this order
EXCLUDED = [0, 1, 252, 253, 259, 0xFFFF]
KEPT = [2, 10, 40, 44, 48, 50, 70, 72, 80, 99, 251]
BEAMS, SPARSE_BEAMS, AZIMUTHS = 8, 4, 96       # scan 1 of every sequence is sparse: shorter than num_points / 10 after the filters
GROUND = 14000                                 # map clutter points besides the scans


def make_scan(g, seed, beams=BEAMS):
    """(n, 4) float32 x, y, z, remission and uint32 labels of one scan, kept clear of the filters' boundaries"""
    from lidiff_b200.synth import synthetic_scan
    xyz = synthetic_scan(seed, beams=beams, azimuths=AZIMUTHS)
    def shell(k, lo, hi):
        d = g.normal(size=(k, 3))
        return d / np.linalg.norm(d, axis=1, keepdims=True) * g.uniform(lo, hi, (k, 1))
    low = np.concatenate([g.uniform(-30, 30, (80, 2)), g.uniform(-5.0, -3.0, (80, 1))], 1)
    pts = np.concatenate([xyz, shell(60, 2.5, 4.5), shell(40, 45.0, 60.0), low])
    pts = pts[g.permutation(pts.shape[0])]
    d = np.linalg.norm(pts, axis=1)
    ok = (np.abs(d - 3.5) >= GEN_MARGIN) & (np.abs(d - MAX_RANGE) >= GEN_MARGIN) & (np.abs(pts[:, 2] + 4.0) >= GEN_MARGIN)
    pts = pts[ok]
    rows = np.concatenate([pts, g.uniform(0, 1, (pts.shape[0], 1))], 1).astype(np.float32)
    rows[5] = [np.nan, 1.0, 1.0, 0.5]
    rows[17] = [np.inf, 2.0, 0.0, 0.5]
    cls = np.where(g.uniform(size=rows.shape[0]) < 0.25, g.choice(EXCLUDED, rows.shape[0]), g.choice(KEPT, rows.shape[0]))
    lab = (cls.astype(np.uint32) | (g.integers(0, 1 << 16, rows.shape[0]).astype(np.uint32) << 16)).astype(np.uint32)
    lab[5] = lab[17] = 40
    return rows, lab


def write_sequence(seq_dir, n_scans, seed):
    from lidiff_b200.kitti import load_poses
    from make_map_goldens import TR, lidar_pose
    os.makedirs(os.path.join(seq_dir, "velodyne"), exist_ok=True)
    os.makedirs(os.path.join(seq_dir, "labels"), exist_ok=True)
    g = np.random.default_rng(seed)
    with open(os.path.join(seq_dir, "calib.txt"), "w") as f:
        f.write("P0: " + " ".join(["0"] * 12) + "\n")
        f.write("Tr: " + " ".join(f"{v:.12e}" for v in TR[:3].reshape(-1)) + "\n")
    with open(os.path.join(seq_dir, "poses.txt"), "w") as f:
        for b in range(n_scans):
            f.write(" ".join(f"{v:.12e}" for v in (TR @ lidar_pose(b) @ np.linalg.inv(TR))[:3].reshape(-1)) + "\n")
    poses = load_poses(os.path.join(seq_dir, "calib.txt"), os.path.join(seq_dir, "poses.txt"))
    world = []
    for b in range(n_scans):
        rows, lab = make_scan(g, seed * 10 + b, SPARSE_BEAMS if b == 1 else BEAMS)
        rows.tofile(os.path.join(seq_dir, "velodyne", f"{b:06d}.bin"))
        lab.tofile(os.path.join(seq_dir, "labels", f"{b:06d}.label"))
        fin = np.isfinite(rows[:, :3]).all(1)
        world.append(rows[fin, :3].astype(np.float64) @ poses[b][:3, :3].T + poses[b][:3, 3])
    ground = np.concatenate([g.uniform(-70, 75, (GROUND, 2)), g.uniform(-5.0, 1.0, (GROUND, 1))], 1)
    m = np.concatenate(world + [ground]).astype(np.float32)
    ok = np.ones(m.shape[0], bool)
    for pose in poses:
        d = np.sqrt(((m.astype(np.float64) - pose[:3, 3]) ** 2).sum(1))
        z = (np.concatenate([m, np.ones((m.shape[0], 1))], 1) @ np.linalg.inv(pose).T)[:, 2]
        ok &= (np.abs(d - MAX_RANGE) >= GEN_MARGIN) & (np.abs(z + 4.0) >= GEN_MARGIN)
    np.save(os.path.join(seq_dir, "map_clean.npy"), m[ok])


def make_dataset(root, seed=SEED):
    """root/dataset/sequences/{00, 01, 08}: scans, labels, calib.txt, poses.txt and map_clean.npy"""
    for i, (seq, n) in enumerate(SEQUENCES.items()):
        write_sequence(os.path.join(root, "dataset", "sequences", seq), n, seed * 100 + i)
    return root


def split_seqs(split):
    return TRAIN if split == "train" else VALIDATION


def record_key(split, k, what):
    return f"{split}_{k}_{what}"


def _cell_margin(p, origin, voxel):
    q = (np.asarray(p, dtype=np.float64) - origin) / voxel
    return (np.abs(q - np.round(q)) * voxel).min() if len(q) else np.inf


def main(ref):
    import importlib
    import torch
    import lidiff_b200.shims as sh
    from oracle.pipeline import farthest_point_sample
    sh.install()
    sys.modules.setdefault("hdbscan", types.ModuleType("hdbscan"))
    mpl = sys.modules.setdefault("matplotlib", types.ModuleType("matplotlib"))
    plt = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot = plt
    sys.modules["matplotlib.pyplot"] = plt
    import open3d as o3d
    from open3d import geometry as G

    def fps(self, n):
        return G.PointCloud(np.asarray(self.points)[farthest_point_sample(np.asarray(self.points), int(n))])
    G.PointCloud.farthest_point_down_sample = fps

    create, included = G.VoxelGrid.create_from_point_cloud, G.VoxelGrid.check_if_included
    worst = {"cell": np.inf}

    def create_checked(inp, voxel_size):
        g = create(inp, voxel_size)
        worst["cell"] = min(worst["cell"], _cell_margin(np.asarray(inp.points), g.origin, g.voxel_size))
        return g

    def included_checked(self, queries):
        worst["cell"] = min(worst["cell"], _cell_margin(np.asarray(queries), self.origin, self.voxel_size))
        return included(self, queries)
    G.VoxelGrid.create_from_point_cloud = staticmethod(create_checked)
    G.VoxelGrid.check_if_included = included_checked
    assert o3d.geometry.VoxelGrid is G.VoxelGrid

    sys.path.insert(0, ref)
    for k in [k for k in sys.modules if k == "lidiff" or k.startswith("lidiff.")]:
        sys.modules.pop(k)
    mod = importlib.import_module("lidiff.datasets.dataloader.SemanticKITTITemporal")
    out = {"seed": np.array(SEED), "num_points": np.array(NUM_POINTS), "max_range": np.array(MAX_RANGE)}
    with tempfile.TemporaryDirectory() as root:
        make_dataset(root)
        for split, indices in RECORD.items():
            ds = mod.TemporalKITTISet(root, split_seqs(split), split, RESOLUTION, NUM_POINTS, MAX_RANGE)
            for path in ds.points_datapath:          # the recorded range / height decisions are clear of their boundaries
                p = np.fromfile(path, dtype=np.float32).reshape(-1, 4)[:, :3].astype(np.float64)
                p = p[np.isfinite(p).all(1)]
                d = np.sqrt((p ** 2).sum(1))
                assert min(np.abs(d - 3.5).min(), np.abs(d - MAX_RANGE).min(), np.abs(p[:, 2] + 4).min()) >= CHECK_MARGIN, path
            np.random.seed(SEED)
            torch.manual_seed(SEED)
            for k, i in enumerate(indices):
                p_full, mean, std, p_part, fname = ds[i]
                out[record_key(split, k, "index")] = np.array(i)
                out[record_key(split, k, "pcd_full")] = p_full.numpy()
                out[record_key(split, k, "mean")] = mean.numpy()
                out[record_key(split, k, "std")] = std.numpy()
                out[record_key(split, k, "pcd_part")] = p_part.numpy()
                out[record_key(split, k, "filename")] = np.array("/".join(fname.split("/")[-3:]))
    assert worst["cell"] >= CELL_MARGIN, f"a point lies {worst['cell']:.3g} m from a viewpoint cell face: choose another SEED"
    np.savez_compressed(os.path.join(HERE, "samples_reference.npz"), **out)
    print({k: v.shape for k, v in out.items() if v.ndim}, "closest cell face", worst["cell"])


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
