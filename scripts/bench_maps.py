#!/usr/bin/env python
"""Ground-truth map building (lidiff_b200.maps / tools.map_from_scans) on a seeded synthetic sequence of ~131 k-point scans with a
moving, turning pose.  Reports the device time per scan (CUDA events around MapBuilder.add_scan), the wall time of the whole
sequence through the CLI's reader (files in a temporary directory), and, in the same run on the same GPU, the reference's algorithm
(concatenate the scan to the map, then de-duplicate the whole map again with torch: unique + first index) for the first
--ref-scans scans, with both maps compared.  Prints one JSON line.

    python scripts/bench_maps.py [--scans 300] [--ref-scans 60] [--device cuda:0]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_eval import gpu_card                      # noqa: E402

VS = 0.1


def pose_of(b):
    a = 0.01 * b
    return np.array([[np.cos(a), -np.sin(a), 0.0, 0.8 * b], [np.sin(a), np.cos(a), 0.0, 0.1 * b], [0, 0, 1.0, 0.0], [0, 0, 0, 1.0]])


def write_sequence(seq, n_scans, seed=0):
    """velodyne/*.bin (64 x 2048 synthetic scans + remission), labels/*.label (10 % moving), poses.txt without calib.txt"""
    from lidiff_b200.synth import synthetic_scan
    os.makedirs(os.path.join(seq, "velodyne"))
    os.makedirs(os.path.join(seq, "labels"))
    g = np.random.default_rng(seed)
    with open(os.path.join(seq, "poses.txt"), "w") as f:
        for b in range(n_scans):
            f.write(" ".join(f"{v:.12e}" for v in pose_of(b)[:3].reshape(-1)) + "\n")
            xyz = synthetic_scan(seed + b % 16)                          # 16 distinct scenes, re-seen from new poses
            np.concatenate([xyz, g.uniform(0, 1, (xyz.shape[0], 1))], 1).astype(np.float32).tofile(
                os.path.join(seq, "velodyne", f"{b:06d}.bin"))
            lab = np.where(g.uniform(size=xyz.shape[0]) < 0.1, 252, 40).astype(np.uint32)
            lab.tofile(os.path.join(seq, "labels", f"{b:06d}.label"))


def reference_algorithm(scans, device):
    """lidiff/map_from_scans.py:64-92 on torch: per scan filter, transform (the same arithmetic order as lb2_map_scan, so the maps
    can be compared bit for bit), concatenate, then floor(map / voxel) and keep the first occurrence of every voxel of the whole map"""
    map_points = torch.empty((0, 3), device=device)
    times = []
    for pts, lab, pose in scans:
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        p = torch.from_numpy(pts).to(device)
        lab = torch.from_numpy(lab.view(np.int32)).to(device) & 0xFFFF
        start.record()
        p = p[(lab < 252) & (lab > 1)]
        p = p[torch.sqrt(((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]) + p[:, 3] * p[:, 3]) > 3.5]
        m = torch.from_numpy(pose[:3, :4].astype(np.float32)).to(device)
        w = torch.stack([((m[k, 0] * p[:, 0] + m[k, 1] * p[:, 1]) + m[k, 2] * p[:, 2]) + m[k, 3] for k in range(3)], 1)
        map_points = torch.cat((map_points, w), 0)
        c = torch.floor(map_points / VS).to(torch.int64)
        _, inv = torch.unique(c, dim=0, return_inverse=True)
        first = torch.full((int(inv.max()) + 1,), c.shape[0], dtype=torch.long, device=device)
        first.scatter_reduce_(0, inv, torch.arange(c.shape[0], device=device), "amin")
        map_points = map_points[torch.sort(first).values]
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
    return map_points, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=300)
    ap.add_argument("--ref-scans", type=int, default=60)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    device = torch.device(args.device)
    torch.cuda.set_device(device)
    from lidiff_b200 import kitti
    from lidiff_b200.maps import MapBuilder
    from lidiff_b200.tools.map_from_scans import build_sequence_map, sequence_scans
    with tempfile.TemporaryDirectory() as root:
        seq = os.path.join(root, "00")
        write_sequence(seq, args.scans)
        pairs = sequence_scans(seq)
        build_sequence_map(seq, VS, 1, device)                                       # untimed: module load, allocator, page cache
        torch.cuda.synchronize()
        t0 = time.time()
        full = build_sequence_map(seq, VS, 1, device)
        wall = time.time() - t0

        scans = [(kitti.read_scan(p), kitti.read_labels(kitti.label_path(p)), pose) for pose, p in pairs]
        mb = MapBuilder(VS, 1, device, initial_capacity=1 << 24)
        per_scan = []
        for pts, lab, pose in scans:
            tp, tl = torch.from_numpy(pts).to(device), torch.from_numpy(lab.view(np.int32)).to(device)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            mb.add_scan(tp, tl, pose)
            end.record()
            torch.cuda.synchronize()
            per_scan.append(start.elapsed_time(end))
        assert mb.points().cpu().numpy().tobytes() == full.tobytes()

        k = min(args.ref_scans, len(scans))
        reference_algorithm(scans[:2], device)                                       # untimed: first calls of torch.unique & co.
        ref_map, ref_times = reference_algorithm(scans[:k], device)
        mk = MapBuilder(VS, 1, device)
        for pts, lab, pose in scans[:k]:
            mk.add_scan(pts, lab, pose)
        same = mk.points().cpu().numpy().tobytes() == ref_map.cpu().numpy().tobytes()
    out = {"what": "ground-truth map of a synthetic sequence (64 x 2048-point scans, 0.1 m voxels, div_mode 1)",
           "card": gpu_card(device.index or 0), "scans": len(scans), "points_per_scan": int(scans[0][0].shape[0]),
           "map_rows": int(full.shape[0]),
           "device_ms_per_scan": {"median": round(statistics.median(per_scan), 3), "max": round(max(per_scan), 3)},
           "device_note": "CUDA events around MapBuilder.add_scan of a scan already on the device (a memset, 4 kernels and the "
                          "8-byte read-back of the row count)",
           "sequence_wall_s": round(wall, 3),
           "sequence_wall_note": "build_sequence_map incl. file reads on the reader thread into pinned buffers; the files were just "
                                 "written, so they come from the page cache",
           "reference_algorithm": {"scans": k, "device_ms_first_scan": round(ref_times[0], 3), "device_ms_last_scan": round(ref_times[-1], 3),
                                   "device_ms_total": round(sum(ref_times), 1), "map_rows": int(ref_map.shape[0]), "same_map": same},
           "streaming_ms_total_first_k": round(sum(per_scan[:k]), 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
