#!/usr/bin/env python
"""Does completing several scans per denoising loop raise scans/s?  For each batch size B (default 1, 2, 3; B = 4 does not fit in 80 GB), at the benchmark's
configuration (180 000 points per scan, 50 steps, seeded random weights with calibrated BatchNorm, synthetic KITTI-shaped scans):

  * ms per denoising step of the fused engine (DenoiseEngine(batch=B).advance, CUDA graphs as in use) and the loop's scans/s;
  * whole-scan scans/s of DiffCompletion.complete_scans on raw scans (preprocessing with farthest point sampling, the loop,
    postprocess, refinement, offsets, results to the host);
  * farthest point sampling of the B raw scans: the single-scan kernel (k_fps_coop) B times against the cluster kernel once;
  * peak device memory.
The batch sizes are measured in alternating order over --reps rounds.  Prints one JSON line per round and a summary line.

    python scripts/bench_batch.py [--batches 1,2,3] [--reps 3] [--steps 50] [--out results/bench_batch.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_POINTS = 180000


def gpu_state(index):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), [c.strip() for c in r.stdout.strip().split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(index), "power.limit": "unavailable"}


def timed(fn, reps=1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps, out


def measure(pipe, raws, B, steps, dev):
    from lidiff_b200.preprocess import farthest_point_sample, farthest_point_sample_batched
    scans = raws[:B]
    n_s = N_POINTS // 10
    pts = [torch.tensor(r, device=dev) for r in scans]
    fps_single, _ = timed(lambda: [farthest_point_sample(p, n_s) for p in pts])
    fps_batched, _ = timed(lambda: farthest_point_sample_batched(pts, n_s))
    pipe._engine = None                                                   # measure the engine of this B from an empty device
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    x_init = pipe.preprocess_scans(scans) if B > 1 else pipe.preprocess_scan(scans[0])
    eng = pipe.engine(B)
    st = eng.start(x_init, x_init + torch.randn(x_init.shape, device=dev), fresh=True)
    for _ in range(3):                                                    # eager step + graph captures
        eng.advance(st, torch.randn((B * N_POINTS, 3), device=dev))
    noise = torch.randn((B * N_POINTS, 3), device=dev)
    ms_loop, _ = timed(lambda: eng.advance(st, noise), steps)
    whole, _ = timed(lambda: pipe.complete_scans(scans, fresh=True))
    return {"B": B, "ms_per_step": ms_loop, "loop_scans_per_s": B * 1e3 / (ms_loop * eng.T), "whole_ms": whole,
            "whole_scans_per_s": B * 1e3 / whole, "fps_single_xB_ms": fps_single, "fps_batched_ms": fps_batched,
            "peak_mem_gib": torch.cuda.max_memory_allocated(dev) / 2 ** 30,
            "peak_bytes_per_row": (torch.cuda.max_memory_allocated(dev) - base) / (B * N_POINTS), "rows": B * N_POINTS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,2,3")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import build_pipeline
    from lidiff_b200.synth import range_filter, synthetic_scan
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    batches = [int(b) for b in args.batches.split(",")]
    raws = [range_filter(synthetic_scan(s)) for s in range(max(batches))]
    calib = torch.tensor(raws[0], device=dev)
    from lidiff_b200.preprocess import farthest_point_sample
    calib = calib[farthest_point_sample(calib, N_POINTS // 10)].repeat(10, 1)
    pipe = build_pipeline(dev, calib)
    state = gpu_state(0)
    rows = []
    for r in range(args.reps):
        order = batches if r % 2 == 0 else batches[::-1]
        for B in order:
            torch.manual_seed(r)
            m = measure(pipe, raws, B, args.steps, dev)
            m["round"] = r
            rows.append(m)
            print(json.dumps(m), flush=True)
    summary = {"gpu": state, "scan_points": [int(r.shape[0]) for r in raws], "n_points": N_POINTS, "steps_timed": args.steps}
    for B in batches:
        mine = [m for m in rows if m["B"] == B]
        summary[f"B{B}"] = {k: statistics.median(m[k] for m in mine) for k in mine[0] if k not in ("B", "round", "rows")}
        summary[f"B{B}"]["spread_ms_per_step"] = [min(m["ms_per_step"] for m in mine), max(m["ms_per_step"] for m in mine)]
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"rounds": rows, "summary": summary}, f, indent=1)


if __name__ == "__main__":
    main()
