"""A synthetic sequence for the `eval_path --voxels / --ssc` tests: the KITTI-style sequence of tests/eval_sequence.py with 11 scans,
scene-completion grid predictions for every 5th scan (`.label`, and one packed `.bin`), the dataset's ground-truth grids
`voxels/<stem>.label` + `.invalid` for those scans, and the same scored scans as a sequence of their own with `.ply` predictions
of the grids' voxel centres (fp64 `double x y z`, so no rounding comes in) for the existing point path."""
import os
import shutil

import numpy as np

import ssc_reference as SR
from eval_sequence import make_sequence
from lidiff_b200.synth import read_ply_xyz
from lidiff_b200.tools.diff_completion_pipeline import write_ply

SCORED = (0, 5, 10)


def make_voxel_sequence(root, n_scans=11, seed=0):
    """(sequence dir, grid prediction dir, sequence of the scored scans, its .ply prediction dir)"""
    seq, pred = make_sequence(str(root), n_scans=n_scans, seed=seed)
    g = np.random.default_rng(seed + 1)
    grids, sub, plys = (os.path.join(str(root), d) for d in ("grids", "sub", "sub_pred"))
    for d in (grids, os.path.join(seq, "voxels"), os.path.join(sub, "velodyne"), plys):
        os.makedirs(d, exist_ok=True)
    poses = open(os.path.join(seq, "poses.txt")).read().splitlines()
    with open(os.path.join(sub, "poses.txt"), "w") as f:
        f.write("\n".join(poses[b] for b in SCORED) + "\n")
    shutil.copy(os.path.join(seq, "calib.txt"), sub)
    shutil.copy(os.path.join(seq, "map_clean.npy"), sub)
    for j, b in enumerate(SCORED):
        stem = f"{b:06d}"
        occ = SR.unpack(SR.voxelize(read_ply_xyz(os.path.join(pred, f"{stem}.ply")))[0])
        if b == 5:
            SR.pack(occ).tofile(os.path.join(grids, f"{stem}.bin"))
        else:
            lab = np.where(occ, g.choice([1, 40, 44, 254, 256], occ.shape[0]), 0).astype("<u2")
            lab[~occ & (g.random(occ.shape[0]) < 0.01)] = 255          # ignored voxels are not predictions
            lab.tofile(os.path.join(grids, f"{stem}.label"))
        write_ply(os.path.join(plys, f"{j:06d}.ply"), SR.centres(occ))
        shutil.copy(os.path.join(seq, "velodyne", f"{stem}.bin"), os.path.join(sub, "velodyne", f"{j:06d}.bin"))
        scan = np.fromfile(os.path.join(seq, "velodyne", f"{stem}.bin"), np.float32).reshape(-1, 4)[:, :3].astype(np.float64)
        gt = SR.unpack(SR.voxelize(scan)[0])
        gt_lab = np.where(gt, 40, 0).astype("<u2")
        gt_lab[g.random(gt.shape[0]) < 0.02] = 255
        gt_lab.tofile(os.path.join(seq, "voxels", f"{stem}.label"))
        SR.pack(g.random(gt.shape[0]) < 0.05).tofile(os.path.join(seq, "voxels", f"{stem}.invalid"))
    return seq, grids, sub, plys
