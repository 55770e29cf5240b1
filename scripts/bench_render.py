#!/usr/bin/env python
"""Time of a point-cloud image (lidiff_b200.render) at 1920x1080 and point sizes 1 and 5, on a cloud shaped like a refined
completion (1.02 M points, tests/normals_oracle.refined_like) and on a 180 000-point completion (a synthetic scan with 6 % of its
points jittered around it): the key-buffer fill, the splat (lb2_render_splat) and the shade (lb2_render_shade), each as the mean
of back-to-back launches between CUDA events, the PNG encode (host clock, zlib level 6), estimate_normals (k = 30, CUDA events), and the numpy restatement of
tests/render_reference.py on the host, all in the same run.  Prints one JSON line.

    python scripts/bench_render.py [--reps 7] [--device cuda:0]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_normals import gpu_state                           # noqa: E402


def completion_like(n=180_000, seed=0):
    from lidiff_b200.synth import synthetic_scan
    g = np.random.default_rng(seed)
    scan = synthetic_scan(seed)
    base = scan[g.choice(scan.shape[0], n, replace=True)]
    return base + g.normal(0.0, 0.05, base.shape)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50, help="back-to-back launches per timed phase")
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    device = torch.device(args.device)
    torch.cuda.set_device(device)
    from lidiff_b200 import _lib
    from lidiff_b200 import render as R
    from lidiff_b200.normals import estimate_normals
    import normals_oracle as O
    import render_reference as rr

    h = _lib.get_handle(device)
    clouds = {"refined_1.02M": O.refined_like(), "completion_180k": completion_like()}
    results = {}
    for name, pts in clouds.items():
        p = torch.as_tensor(pts, device=device)
        cam = R.Camera.fit(pts)
        c = cam.c_struct()
        z_lo, z_hi = float(pts[:, 2].min()), float(pts[:, 2].max())
        nrm = estimate_normals(p, knn=30, device=device)
        t_nrm = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            estimate_normals(p, knn=30, device=device)
            e1.record()
            torch.cuda.synchronize()
            t_nrm.append(e0.elapsed_time(e1))
        row = {"n_points": int(pts.shape[0]), "estimate_normals_ms": round(statistics.median(t_nrm), 3)}
        for s in (1, 5):
            keys = torch.empty(cam.width * cam.height, dtype=torch.int64, device=device)
            rgb = torch.empty((cam.height, cam.width, 3), dtype=torch.uint8, device=device)
            for _ in range(2):                                  # warm-up
                keys.fill_(-1)
                h.render_splat(p, c, s, keys)
                h.render_shade(keys, p, nrm, None, z_lo, z_hi, c, rgb)
            fill, splat, shade, png = [], [], [], []
            for _ in range(args.reps):
                # each phase is launched `launches` times back to back between two events, so the host's launch gap is hidden
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                ev[0].record()
                for _ in range(args.launches):
                    keys.fill_(-1)
                ev[1].record()
                for _ in range(args.launches):                   # a fill before every splat, so every splat starts from the background
                    keys.fill_(-1)
                    h.render_splat(p, c, s, keys)
                ev[2].record()
                for _ in range(args.launches):
                    h.render_shade(keys, p, nrm, None, z_lo, z_hi, c, rgb)
                ev[3].record()
                torch.cuda.synchronize()
                fill.append(ev[0].elapsed_time(ev[1]) / args.launches)
                splat.append((ev[1].elapsed_time(ev[2]) - ev[0].elapsed_time(ev[1])) / args.launches)
                shade.append(ev[2].elapsed_time(ev[3]) / args.launches)
                t0 = time.time()
                R.encode_png(rgb)
                png.append(1e3 * (time.time() - t0))
            keys.fill_(-1)
            h.render_splat(p, c, s, keys)
            h.render_shade(keys, p, nrm, None, z_lo, z_hi, c, rgb)
            keys_gpu, rgb_gpu = keys.cpu().numpy().view(np.uint64), rgb.cpu().numpy()
            t0 = time.time()
            ref_keys, ref_rgb = rr.render(pts, cam, normals=nrm.cpu().numpy(), point_size=s, z_range=(z_lo, z_hi))
            t_ref = 1e3 * (time.time() - t0)
            covered = int((keys_gpu != rr.EMPTY).sum())
            row[f"point_size_{s}"] = {
                "key_fill_ms": round(statistics.median(fill), 4), "splat_ms": round(statistics.median(splat), 4),
                "shade_ms": round(statistics.median(shade), 4),
                "png_encode_ms": round(statistics.median(png), 1), "numpy_restatement_ms": round(t_ref, 1),
                "covered_pixels": covered, "bit_exact_vs_restatement": bool(np.array_equal(keys_gpu, ref_keys) and np.array_equal(rgb_gpu, ref_rgb))}
        results[name] = row
    state = gpu_state(device.index or 0)
    print(json.dumps({"what": "point-cloud image at 1920x1080 (lidiff_b200.render): splat, shade, PNG encode, estimate_normals",
                      "card": state, "reps": args.reps, "results": results,
                      "launches": args.launches,
                      "note": "median over reps of the mean over `launches` back-to-back launches (CUDA events): key fill; splat = "
                              "(fill + splat) - fill; shade; png_encode from the host clock "
                              "(device-to-host copy + zlib); numpy restatement: one host run, one core"}))


if __name__ == "__main__":
    main()
