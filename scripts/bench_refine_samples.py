#!/usr/bin/env python
"""The refinement network's samples (lidiff_b200.datasets_refine.TemporalKITTISet) at the reference's settings: windows of 40 scans,
num_points 180 000, on a seeded synthetic sequence of ~115 k-point scans (files in a temporary directory), validation and train split.
Reports, per sample (after one untimed sample): samples/s, and its split into host random draws (numpy's randn over every row and
torch's two randperms), file reads, and device time of the three sample kernels by CUDA events; the per-batch loss time (refinement
MinkUNet forward with seeded random weights + Chamfer distance, 1 080 000 refined vs 360 000 ground-truth points, B = 1); and, in
the same run, the seconds of a numpy restatement of one validation sample on the host (written here; the Chamfer loss is not part
of it).  Prints one JSON line with the card name and power limit.

    python scripts/bench_refine_samples.py [--scans 40] [--samples 3] [--host 1] [--device cuda:0]
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

NUM_POINTS, WINDOW, AZIMUTHS = 180000, 40, 1800


def write_sequence(seq, n_scans, seed=0):
    """velodyne/*.bin (64 x 1800 synthetic scans), labels/*.label (10 % moving), poses.txt (no calib.txt)"""
    from lidiff_b200.synth import synthetic_scan
    os.makedirs(os.path.join(seq, "velodyne"))
    os.makedirs(os.path.join(seq, "labels"))
    g = np.random.default_rng(seed)
    with open(os.path.join(seq, "poses.txt"), "w") as f:
        for b in range(n_scans):
            a = 0.01 * b
            pose = np.array([[np.cos(a), -np.sin(a), 0.0, 0.8 * b], [np.sin(a), np.cos(a), 0.0, 0.1 * b], [0, 0, 1.0, 0.0]])
            f.write(" ".join(f"{v:.12e}" for v in pose.reshape(-1)) + "\n")
            xyz = synthetic_scan(seed + b, azimuths=AZIMUTHS)
            np.concatenate([xyz, g.uniform(0, 1, (xyz.shape[0], 1))], 1).astype(np.float32).tofile(
                os.path.join(seq, "velodyne", f"{b:06d}.bin"))
            np.where(g.uniform(size=xyz.shape[0]) < 0.1, 252, 40).astype(np.uint32).tofile(os.path.join(seq, "labels", f"{b:06d}.label"))


def host_sample(ds, index):
    """the reference's validation __getitem__ restated in numpy: aggregate_pcds, jitter, first occurrence per 0.1 m voxel, the 50 m
    tests, randperm / repeat / truncate, mean and std"""
    window = ds.points_datapath[index]
    poses = ds.seq_poses[window[0].split("/")[-3]]
    t_frame = len(window) // 2
    full, part = [], None
    for t, path in enumerate(window):
        p = np.fromfile(path, dtype=np.float32).reshape(-1, 4)[:, :3]
        lab = np.fromfile(path.replace("velodyne", "labels").replace(".bin", ".label"), dtype=np.uint32) & 0xFFFF
        p = p[lab < 252]
        p = p[np.sqrt((p ** 2).sum(-1)) > 3.5]
        h = np.hstack((p, np.ones_like(p[:, :1])))
        p = np.sum(np.expand_dims(h, 2) * poses[int(os.path.basename(path).split(".")[0])].T, axis=1)[:, :3]
        if t == t_frame:
            part = p
        else:
            full.append(p)
    undo = np.linalg.inv(poses[int(os.path.basename(window[-1]).split(".")[0])]).T
    undo_t = lambda q: np.sum(np.expand_dims(np.hstack((q, np.ones_like(q[:, :1]))), 2) * undo, axis=1)[:, :3]
    p_concat = np.concatenate((undo_t(np.concatenate(full)), undo_t(part)))
    p_noise = p_concat + np.clip(0.2 * np.random.randn(1, *p_concat.shape), -0.3, 0.3)[0]
    p_noise = p_noise[np.sqrt((p_noise ** 2).sum(-1)) < 50.0]
    q = np.floor(p_concat / 0.1).astype(np.int64)
    _, first = np.unique(q, axis=0, return_index=True)
    p_full = p_concat[np.sort(first)]
    p_full = p_full[np.sqrt((p_full ** 2).sum(-1)) < 50.0]
    p_full = p_full[torch.randperm(p_full.shape[0]).numpy()]
    p_full = p_full.repeat(int(np.ceil(2 * NUM_POINTS / p_full.shape[0])), 0)[: 2 * NUM_POINTS]
    p_noise = p_noise[torch.randperm(p_noise.shape[0]).numpy()]
    p_noise = p_noise.repeat(int(np.ceil(NUM_POINTS / p_noise.shape[0])), 0)[:NUM_POINTS]
    return p_full, p_full.mean(0), p_full.std(0, ddof=1), p_noise


class Timers:
    """accumulates host seconds of the random draws and file reads and CUDA-event milliseconds of the sample kernels"""

    def __init__(self, ds):
        from lidiff_b200 import datasets_refine as R
        self.t = {"rng_s": 0.0, "read_s": 0.0}
        self.events = []
        self.patches = []
        for mod, name, key in ((np.random, "randn", "rng_s"), (torch, "randperm", "rng_s"), (R, "read_scan", "read_s"),
                               (R, "read_labels", "read_s")):
            self._wrap_host(mod, name, key)
        for name in ("aggregate_window", "jitter_filter", "voxel_first_f64"):
            self._wrap_device(ds.h, name)

    def _wrap_host(self, mod, name, key):
        f = getattr(mod, name)
        def g(*a, **k):
            t0 = time.perf_counter()
            try:
                return f(*a, **k)
            finally:
                self.t[key] += time.perf_counter() - t0
        setattr(mod, name, g)
        self.patches.append((mod, name, f))

    def _wrap_device(self, h, name):
        f = getattr(h, name)
        def g(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f(*a, **k)
            e1.record()
            self.events.append((e0, e1))
        setattr(h, name, g)
        self.patches.append((h, name, None))

    def reset(self):
        self.t = {"rng_s": 0.0, "read_s": 0.0}
        self.events = []

    def device_ms(self):
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self.events)

    def restore(self):
        for mod, name, f in reversed(self.patches):
            if f is None:
                delattr(mod, name)
            else:
                setattr(mod, name, f)


def loss_bench(dev, batch, reps):
    from lidiff_b200.tools.test_refine import load_refine_net, refine_batch
    net = load_refine_net(None, 6, dev, random_weights=True)
    refine_batch(net, batch, 0.05, 6, dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        _, loss = refine_batch(net, batch, 0.05, 6, dev)
    loss.item()
    return 1e3 * (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=WINDOW)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--loss-reps", type=int, default=3)
    ap.add_argument("--host", type=int, default=1, help="host samples to time (0: skip)")
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args()
    from lidiff_b200.datasets_refine import SparseSegmentCollation, TemporalKITTISet
    dev = torch.device(a.device)
    torch.cuda.set_device(dev)
    res = {"bench": "refine_samples", "num_points": NUM_POINTS, "scan_window": WINDOW, "card": gpu_card(dev.index or 0),
           "host_threads": torch.get_num_threads()}
    with tempfile.TemporaryDirectory() as root:
        write_sequence(os.path.join(root, "dataset", "sequences", "00"), a.scans)
        for split in ("validation", "train"):
            ds = TemporalKITTISet(root, WINDOW, ["00"], split, 0.05, NUM_POINTS, "refine", device=dev)
            np.random.seed(0)
            torch.manual_seed(0)
            item = ds[0]
            res["window_rows"] = int(ds.aggregate(0).shape[0])
            tm = Timers(ds)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for k in range(a.samples):
                item = ds[k % len(ds)]
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) / a.samples
            res[f"{split}_samples_per_s"] = round(1 / dt, 3)
            res[f"{split}_s_per_sample"] = round(dt, 3)
            res[f"{split}_host_rng_s"] = round(tm.t["rng_s"] / a.samples, 3)
            res[f"{split}_file_read_s"] = round(tm.t["read_s"] / a.samples, 3)
            res[f"{split}_device_kernels_ms"] = round(tm.device_ms() / a.samples, 2)
            tm.restore()
            assert item[0].shape == (2 * NUM_POINTS, 3) and item[3].shape == (NUM_POINTS, 3)
            if split == "validation":
                res["loss_ms_per_batch"] = round(loss_bench(dev, SparseSegmentCollation("refine")([item]), a.loss_reps), 1)
                if a.host:
                    t0 = time.perf_counter()
                    for i in range(a.host):
                        host_sample(ds, i % len(ds))
                    res["host_restatement_s_per_sample"] = round((time.perf_counter() - t0) / a.host, 2)
            del ds
    print(json.dumps(res))


if __name__ == "__main__":
    main()
