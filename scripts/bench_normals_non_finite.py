#!/usr/bin/env python
"""Time of lidiff_b200.normals.estimate_normals (k = 30: tree build + k-NN + normals) on the 1.02 M-point refined-completion-shaped
cloud of tests/normals_oracle.py, with and without four rows that hold a NaN or infinite coordinate (+inf, -inf, an all-NaN row and
a NaN with the sign bit set), alternating the two clouds, by CUDA events around each call.  Such rows must not shape the tree
(csrc/metrics.cu), so both times should be the same.  Prints one JSON line.

    python scripts/bench_normals_non_finite.py [--reps 10] [--device cuda:0]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_normals import gpu_state                            # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    device = torch.device(args.device)
    torch.cuda.set_device(device)
    from lidiff_b200.normals import estimate_normals
    import normals_oracle as O

    fin = O.refined_like()
    bad = np.array([[np.inf, 0.0, 0.0], [0.0, -np.inf, 1.0], [np.nan] * 3, [1.0, np.copysign(np.nan, -1.0), 2.0]])
    pos = np.sort(np.random.default_rng(0).choice(fin.shape[0] + 4, 4, replace=False))
    mixed = np.insert(fin, pos - np.arange(4), bad, axis=0)
    clouds = {"finite": torch.as_tensor(fin, device=device), "with_4_non_finite": torch.as_tensor(mixed, device=device)}
    for p in clouds.values():                                   # warm-up: module load, allocator
        estimate_normals(p, device=device)
    torch.cuda.synchronize()
    ms = {name: [] for name in clouds}
    for _ in range(args.reps):
        for name, p in clouds.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            estimate_normals(p, device=device)
            b.record()
            torch.cuda.synchronize()
            ms[name].append(a.elapsed_time(b))
    print(json.dumps({"what": "estimate_normals(k=30) on a refined-completion-shaped cloud, with and without 4 non-finite rows",
                      "n_points": int(fin.shape[0]), "card": gpu_state(device.index or 0), "reps": args.reps,
                      "ms_median": {k: round(statistics.median(v), 3) for k, v in ms.items()},
                      "ms_min_max": {k: [round(min(v), 3), round(max(v), 3)] for k, v in ms.items()},
                      "note": "CUDA events around the public call (tree build, k-NN, normals, allocations), alternating clouds"}))


if __name__ == "__main__":
    main()
