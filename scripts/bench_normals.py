#!/usr/bin/env python
"""Time of open3d-style point normals (lidiff_b200.normals.estimate_normals, k = 30) on a cloud shaped like a refined completion
(~170 000 points of a synthetic scan with 6 offsets of a few cm around each: 1.02 M points), split into tree build, k-NN and
normals with CUDA events, next to the open3d shim's former GPU path (the bucketed torch `_knn` + batched `torch.linalg.eigh`) and
the numpy restatement of tests/normals_oracle.py on the host cores, all in the same run.  Prints one JSON line.

    python scripts/bench_normals.py [--reps 7] [--device cuda:0]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench import usable_cpus                                  # noqa: E402


def gpu_state(index):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), [c.strip() for c in r.stdout.strip().split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(index), "power.limit": "unavailable"}


def old_shim_path(p64, k=30, batch=65536):
    """the open3d shim's estimate_normals as it ran on a GPU before lb2_pc_normals: fp32 bucketed k-NN, two-pass covariance, eigh
    over batches of `batch` matrices (65 536 in the shim).  Returns (normals, k-NN ms, covariance + eigh ms)."""
    from lidiff_b200.shims.open3d.geometry import _knn
    p = p64.float()
    n = p.shape[0]
    out = torch.zeros((n, 3), dtype=torch.float32, device=p.device)
    torch.cuda.synchronize()
    t0 = time.time()
    _, idx = _knn(p, p, k)
    torch.cuda.synchronize()
    t1 = time.time()
    for a in range(0, n, batch):
        nb = p[idx[a:a + batch]]
        c = nb - nb.mean(1, keepdim=True)
        out[a:a + batch] = torch.linalg.eigh((c.transpose(1, 2) @ c).double())[1][:, :, 0].float()
    torch.cuda.synchronize()
    return out, 1e3 * (t1 - t0), 1e3 * (time.time() - t1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    device = torch.device(args.device)
    torch.cuda.set_device(device)
    from lidiff_b200 import _lib
    from lidiff_b200.normals import estimate_normals
    import normals_oracle as O

    pts = O.refined_like()
    n, k = pts.shape[0], 30
    h = _lib.get_handle(device)
    p = torch.as_tensor(pts, device=device)
    idx = torch.empty((n, k), dtype=torch.int32, device=device)
    nrm = torch.empty((n, 3), dtype=torch.float64, device=device)
    for _ in range(2):                                          # warm-up: module load, allocator
        h.pc_knn(h.pc_tree(p), n, k, idx)
        h.pc_normals(p, idx, nrm)
    torch.cuda.synchronize()
    phases = {"tree_build": [], "knn": [], "normals": [], "estimate_normals_wall": []}
    for _ in range(args.reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        tree = h.pc_tree(p)
        ev[1].record()
        h.pc_knn(tree, n, k, idx)
        ev[2].record()
        h.pc_normals(p, idx, nrm)
        ev[3].record()
        torch.cuda.synchronize()
        for name, a, b in (("tree_build", 0, 1), ("knn", 1, 2), ("normals", 2, 3)):
            phases[name].append(ev[a].elapsed_time(ev[b]))
        t0 = time.time()
        estimate_normals(p, knn=k, device=device)
        torch.cuda.synchronize()
        phases["estimate_normals_wall"].append(1e3 * (time.time() - t0))
    gpu = {name: round(statistics.median(v), 3) for name, v in phases.items()}
    state = gpu_state(device.index or 0)                       # read right after the timed phase

    new = nrm.cpu().numpy()
    old_runs = {}
    for batch in (65536, 8192):                                 # the shim's batch, then a smaller one if cuSOLVER refuses it
        try:
            old, t_knn, t_eig = old_shim_path(p, k, batch)
        except RuntimeError as e:
            old_runs[f"eigh_batch_{batch}"] = {"error": str(e).split(". ")[0][:300]}
            continue
        old_runs[f"eigh_batch_{batch}"] = {"knn_ms": round(t_knn, 1), "cov_eigh_ms": round(t_eig, 1), "total_ms": round(t_knn + t_eig, 1),
                                           "mean_abs_cos_vs_new": round(float(np.abs((old.double().cpu().numpy() * new).sum(1)).mean()), 6)}
        break

    cores = usable_cpus()
    t0 = time.time()
    ref_idx, _ = O.knn(pts, k)
    t1 = time.time()
    O.normals_from_idx(pts, ref_idx)
    t2 = time.time()
    print(json.dumps({
        "what": "open3d estimate_normals() (KDTreeSearchParamKNN(30), FastEigen3x3) of one refined-completion-shaped cloud",
        "n_points": n, "k": k, "card": state, "reps": args.reps,
        "gpu_ms": gpu, "gpu_ms_note": "median over reps; phases from CUDA events; estimate_normals_wall = host clock of the public call "
                                      "incl. allocation and a device synchronise",
        "old_shim_gpu": old_runs, "old_shim_note": "torch _knn (fp32, chunks of 4096 queries) + two-pass covariance + batched eigh, "
                                                   "one run after the timed phase; host clock with synchronise",
        "cpu_ms": {"knn": round(1e3 * (t1 - t0), 1), "normals": round(1e3 * (t2 - t1), 1)},
        "cpu_note": f"numpy restatement: scipy cKDTree (workers=-1, {cores} usable cores) + numpy covariance and FastEigen3x3 "
                    "(vectorised, one core), one run"}))


if __name__ == "__main__":
    main()
