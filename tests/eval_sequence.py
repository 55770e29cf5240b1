"""A small synthetic KITTI-style sequence for the eval_path tests: velodyne/*.bin scans from lidiff_b200.synth, calib.txt,
poses.txt (moving and turning sensor) and a map_clean.npy built from the scans in the world frame, plus a `.ply` prediction per
scan (the scan with noise, spurious points and points beyond the histogram range)."""
import os

import numpy as np

from lidiff_b200.synth import synthetic_scan
from lidiff_b200.tools.diff_completion_pipeline import write_ply

TR = np.array([[0.0, -1.0, 0.0, 0.1], [0.0, 0.0, -1.0, -0.05], [1.0, 0.0, 0.0, -0.3], [0.0, 0.0, 0.0, 1.0]])   # LiDAR -> camera


def lidar_pose(b):
    a = 0.05 * b
    return np.array([[np.cos(a), -np.sin(a), 0.0, 2.0 * b], [np.sin(a), np.cos(a), 0.0, 0.5 * b], [0, 0, 1.0, 0.0], [0, 0, 0, 1.0]])


def make_sequence(root, n_scans=3, beams=16, azimuths=512, seed=0):
    """writes the sequence under root/seq and the predictions under root/pred/; returns (seq dir, pred dir)"""
    seq, pred = os.path.join(root, "seq"), os.path.join(root, "pred")
    os.makedirs(os.path.join(seq, "velodyne"), exist_ok=True)
    os.makedirs(pred, exist_ok=True)
    g = np.random.default_rng(seed)
    with open(os.path.join(seq, "calib.txt"), "w") as f:
        f.write("P0: " + " ".join(["0"] * 12) + "\n")
        f.write("Tr: " + " ".join(f"{v:.12e}" for v in TR[:3].reshape(-1)) + "\n")
    world = []
    with open(os.path.join(seq, "poses.txt"), "w") as f:
        for b in range(n_scans):
            scan = synthetic_scan(seed + b, beams=beams, azimuths=azimuths)
            rows = np.concatenate([scan, g.uniform(0, 1, (scan.shape[0], 1))], 1).astype(np.float32)
            rows.tofile(os.path.join(seq, "velodyne", f"{b:06d}.bin"))
            p = lidar_pose(b)
            cam = TR @ p @ np.linalg.inv(TR)                   # poses.txt holds camera-frame poses
            f.write(" ".join(f"{v:.12e}" for v in cam[:3].reshape(-1)) + "\n")
            world.append(scan @ p[:3, :3].T + p[:3, 3])
            pts = scan[g.choice(scan.shape[0], scan.shape[0] * 2 // 3, replace=False)] + g.normal(0, 0.05, (scan.shape[0] * 2 // 3, 3))
            extra = np.concatenate([g.uniform(-30, 30, (300, 3)) * [1, 1, 0.1], [[49.5, 0.0, 0.0], [0.0, 0.0, 0.0]]])
            write_ply(os.path.join(pred, f"{b:06d}.ply"), np.concatenate([pts, extra]))
    np.save(os.path.join(seq, "map_clean.npy"), np.concatenate(world))
    return seq, pred
