#!/usr/bin/env python
"""The diffusion network's training / test samples (lidiff_b200.datasets.TemporalKITTISet.batch) at the reference's settings:
180 000 points, batches of 2, the train and the validation split, on a seeded synthetic sequence of 131 k-point scans and a map of
--map-points points (files in a temporary directory).  Reports samples per second of batch() (wall time, the files read and the
sequence map resident on the device, after one untimed batch), and, in the same run, the seconds per sample of the host
restatement of one validation sample: the reference's numpy steps with the oracle's numpy farthest point sampling (oracle/pipeline.py),
which is what the reference's __getitem__ runs on the host cores (open3d's FPS is a C++ loop of the same work).  Prints one JSON line.

    python scripts/bench_samples.py [--map-points 20000000] [--batches 5] [--device cuda:0]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_eval import gpu_card                      # noqa: E402

NUM_POINTS, MAX_RANGE, BATCH = 180000, 50.0, 2


def pose_of(b):
    a = 0.01 * b
    return np.array([[np.cos(a), -np.sin(a), 0.0, 0.8 * b], [np.sin(a), np.cos(a), 0.0, 0.1 * b], [0, 0, 1.0, 0.0], [0, 0, 0, 1.0]])


def write_sequence(seq, n_scans, map_points, seed=0):
    """velodyne/*.bin (64 x 2048 synthetic scans), labels/*.label (10 % moving), poses.txt (no calib.txt), map_clean.npy: the scans
    in the world frame plus uniform ground clutter over +-150 m (float32)"""
    from lidiff_b200.synth import synthetic_scan
    os.makedirs(os.path.join(seq, "velodyne"))
    os.makedirs(os.path.join(seq, "labels"))
    g = np.random.default_rng(seed)
    world = []
    with open(os.path.join(seq, "poses.txt"), "w") as f:
        for b in range(n_scans):
            pose = pose_of(b)
            f.write(" ".join(f"{v:.12e}" for v in pose[:3].reshape(-1)) + "\n")
            xyz = synthetic_scan(seed + b)
            np.concatenate([xyz, g.uniform(0, 1, (xyz.shape[0], 1))], 1).astype(np.float32).tofile(
                os.path.join(seq, "velodyne", f"{b:06d}.bin"))
            np.where(g.uniform(size=xyz.shape[0]) < 0.1, 252, 40).astype(np.uint32).tofile(os.path.join(seq, "labels", f"{b:06d}.label"))
            world.append((xyz @ pose[:3, :3].T + pose[:3, 3]).astype(np.float32))
    k = max(map_points - sum(w.shape[0] for w in world), 0)
    clutter = np.empty((k, 3), np.float32)
    clutter[:, :2] = g.uniform(-150, 150, (k, 2))
    clutter[:, 2] = g.uniform(-3, 3, k)
    np.save(os.path.join(seq, "map_clean.npy"), np.concatenate(world + [clutter]))


def host_sample(ds, index):
    """the reference's __getitem__ for a validation sample in numpy, FPS by the oracle's numpy loop"""
    from lidiff_b200.shims.open3d.geometry import PointCloud, VoxelGrid
    from oracle.pipeline import farthest_point_sample
    path = ds.points_datapath[index]
    p_part = np.fromfile(path, dtype=np.float32).reshape((-1, 4))[:, :3]
    lab = np.fromfile(path.replace("velodyne", "labels").replace(".bin", ".label"), dtype=np.uint32) & 0xFFFF
    p_part = p_part[(lab < 252) & (lab > 1)]
    d = np.sum(p_part ** 2, -1) ** .5
    p_part = p_part[(d < MAX_RANGE) & (d > 3.5)]
    p_part = p_part[p_part[:, 2] > -4.]
    pose = ds.seq_poses[index]
    p_map = ds.host_map
    dist = np.sum((p_map - pose[:-1, -1]) ** 2, -1) ** .5
    p_full = p_map[dist < MAX_RANGE]
    p_full = (np.concatenate((p_full, np.ones((len(p_full), 1))), axis=-1) @ np.linalg.inv(pose).T)[:, :3]
    p_full = p_full[p_full[:, 2] > -4.]
    n_part = int(NUM_POINTS / 10.)
    p_part = p_part.repeat(np.ceil(n_part / p_part.shape[0]), 0)
    grid = VoxelGrid.create_from_point_cloud(PointCloud(p_part), 10.0)
    p_part = torch.tensor(p_part[farthest_point_sample(p_part, n_part)])
    p_full = p_full[np.asarray(grid.check_if_included(p_full))]
    p_full = p_full[torch.randperm(p_full.shape[0])]
    p_full = torch.tensor(p_full.repeat(np.ceil(NUM_POINTS / p_full.shape[0]), 0)[:NUM_POINTS])
    return p_full, p_full.mean(0), p_full.std(0), p_part


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--map-points", type=int, default=20_000_000)
    ap.add_argument("--scans", type=int, default=4)
    ap.add_argument("--batches", type=int, default=5)
    ap.add_argument("--host", type=int, default=1, help="host samples to time (0: skip)")
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args()
    from lidiff_b200.datasets import TemporalKITTISet
    dev = torch.device(a.device)
    torch.cuda.set_device(dev)
    res = {"bench": "samples", "num_points": NUM_POINTS, "batch": BATCH, "card": gpu_card(dev.index or 0)}
    with tempfile.TemporaryDirectory() as root:
        seq = os.path.join(root, "dataset", "sequences", "00")
        write_sequence(seq, a.scans, a.map_points)
        res["map_points"] = int(np.load(os.path.join(seq, "map_clean.npy"), mmap_mode="r").shape[0])
        for split in ("train", "validation"):
            ds = TemporalKITTISet(root, ["00"], split, 0.05, NUM_POINTS, MAX_RANGE, device=dev)
            np.random.seed(0)
            torch.manual_seed(0)
            order = [[(BATCH * k + j) % len(ds) for j in range(BATCH)] for k in range(a.batches + 1)]
            ds.batch(order[0])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for idx in order[1:]:
                b = ds.batch(idx)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            res[f"{split}_samples_per_s"] = round(BATCH * a.batches / dt, 3)
            res[f"{split}_ms_per_batch"] = round(1e3 * dt / a.batches, 2)
            assert b["pcd_full"].shape == (BATCH, NUM_POINTS, 3) and b["pcd_part"].shape == (BATCH, NUM_POINTS // 10, 3)
            if split == "validation" and a.host:
                ds.host_map = np.load(os.path.join(seq, "map_clean.npy"))
                t0 = time.perf_counter()
                for i in range(a.host):
                    host_sample(ds, i % len(ds))
                res["host_s_per_sample"] = round((time.perf_counter() - t0) / a.host, 2)
                res["host_threads"] = torch.get_num_threads()
            del ds
    print(json.dumps(res))


if __name__ == "__main__":
    main()
