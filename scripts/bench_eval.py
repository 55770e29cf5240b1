#!/usr/bin/env python
"""Per-scan time of the evaluation metrics (lidiff_b200.metrics.evaluate_scan) on a scan-sized pair, split by phase with CUDA
events, next to the same evaluation with scipy / numpy on the host cores in the same run.  Prints one JSON line.

    python scripts/bench_eval.py [--reps 5] [--device cuda:0]
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
from bench import usable_cpus                                  # noqa: E402


def eval_pair(seed=0):
    """a scan-sized evaluation pair: ~1.05 M ground-truth points (8 synthetic scans) and ~1.0 M predicted points (6 offsets of
    0.05 m around 170 000 of them, the shape of a refined completion), fp64"""
    from lidiff_b200.synth import synthetic_scan
    g = np.random.default_rng(seed)
    gt = np.concatenate([synthetic_scan(seed + k) for k in range(8)])
    base = gt[g.choice(gt.shape[0], 170_000, replace=False)]
    pred = (base[:, None, :] + g.normal(0.0, 0.05, (base.shape[0], 6, 3))).reshape(-1, 3)
    return gt, pred


def gpu_card(index):
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        name, limit = [c.strip() for c in r.stdout.strip().split(",")[:2]]
        return {"name": name, "power_limit": limit}
    except Exception:
        return {"name": torch.cuda.get_device_name(index), "power_limit": "unavailable"}


def eval_bench(device, reps=5):
    """per-scan evaluation (lidiff_b200.metrics.evaluate_scan: nearest neighbours both ways, PR counts at 100 thresholds,
    occupancy / IoU at 0.5, 0.2, 0.1 m, 3D + BEV JSD) on a ~1 M / ~1 M pair; CUDA events per phase.  Then the same evaluation with
    scipy's cKDTree (all host cores) and numpy (searchsorted + unique for the occupancies, histogramdd for the JSD) in the same run."""
    from scipy.spatial import cKDTree
    from scipy.spatial.distance import jensenshannon
    from lidiff_b200 import metrics as M
    gt_np, pred_np = eval_pair()
    gt, pred = torch.as_tensor(gt_np, device=device), torch.as_tensor(pred_np, device=device)
    M.evaluate_scan(gt, pred, device=device)                                # untimed: module load, allocator
    phases, wall = [], []
    for _ in range(reps):
        ev = {}
        torch.cuda.synchronize()
        t0 = time.time()
        M.evaluate_scan(gt, pred, device=device, events=ev)
        wall.append(1e3 * (time.time() - t0))
        el = lambda a, b: a.elapsed_time(b)
        ph = {"nn_build": sum(el(a, b) for a, b in zip(ev["nn_build"], ev["nn_query"])),
              "nn_query_and_counts": sum(el(a, b) for a, b in zip(ev["nn_query"], ev["nn_end"]))}
        for j, vs in enumerate(M.VOXEL_SIZES):
            stop = ev["jsd"][0] if vs == M.JSD_VOXEL else ev["occupancy_end"][j]
            ph[f"occupancy_iou_{vs}"] = el(ev[f"occupancy_{vs}"][0], stop)
        ph["jsd_3d_bev"] = el(ev["jsd"][0], ev["occupancy_end"][M.VOXEL_SIZES.index(M.JSD_VOXEL)])
        phases.append(ph)
    gpu = {k: round(statistics.median(p[k] for p in phases), 3) for k in phases[0]}
    gpu["total_wall_ms"] = round(statistics.median(wall), 3)

    cores = usable_cpus()
    cpu = {}
    t0 = time.time()
    tg, tp = cKDTree(gt_np), cKDTree(pred_np)
    cpu["nn_build"] = 1e3 * (time.time() - t0)
    t0 = time.time()
    d_pg, _ = tg.query(pred_np, workers=cores)
    d_gp, _ = tp.query(gt_np, workers=cores)
    thr = np.linspace(*M.PR_ARGS)
    np.searchsorted(np.sort(d_pg), thr), np.searchsorted(np.sort(d_gp), thr)
    cpu["nn_query_and_counts"] = 1e3 * (time.time() - t0)
    for vs in M.VOXEL_SIZES:
        t0 = time.time()
        e = M.voxel_edges(vs)
        nb = e.shape[0] - 1
        cells = []
        for x in (gt_np, pred_np):
            b = np.searchsorted(e, x, side="right") - 1
            b[x == e[-1]] = nb - 1
            ok = ((b >= 0) & (b < nb)).all(1)
            cells.append(np.unique((b[ok, 0] * nb + b[ok, 1]) * nb + b[ok, 2]))
        np.intersect1d(cells[0], cells[1], assume_unique=True).shape
        cpu[f"occupancy_iou_{vs}"] = 1e3 * (time.time() - t0)
    t0 = time.time()
    rng = [[-50, 50]] * 3
    hg, hp = np.histogramdd(gt_np, bins=200, range=rng)[0], np.histogramdd(pred_np, bins=200, range=rng)[0]
    jensenshannon((hg / hg.sum()).ravel(), (hp / hp.sum()).ravel())
    bg, bp = np.clip(hg, 0, 1).sum(-1), np.clip(hp, 0, 1).sum(-1)
    jensenshannon((bg / bg.sum()).ravel(), (bp / bp.sum()).ravel())
    cpu["jsd_3d_bev"] = 1e3 * (time.time() - t0)
    cpu = {k: round(v, 1) for k, v in cpu.items()}
    cpu["total_ms"] = round(sum(cpu.values()), 1)
    return {"what": "per-scan evaluation of one (ground truth, completion) pair: exact fp64 1-NN both ways + sums + counts below 100 PR "
                    "thresholds, occupancy and IoU counts at 0.5 / 0.2 / 0.1 m, 3D and BEV Jensen-Shannon distance at 0.5 m",
            "n_gt": int(gt_np.shape[0]), "n_pred": int(pred_np.shape[0]), "card": gpu_card(device.index or 0), "reps": reps,
            "gpu_ms": gpu, "gpu_ms_note": "median over reps; phases from CUDA events, total = host wall clock of evaluate_scan incl. its one synchronisation",
            "cpu_ms": cpu, "cpu_note": f"scipy cKDTree (workers={cores}) and numpy on the host cores, one run"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    device = torch.device(args.device)
    torch.cuda.set_device(device)
    print(json.dumps(eval_bench(device, args.reps)))


if __name__ == "__main__":
    main()
