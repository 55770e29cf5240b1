#!/usr/bin/env python
"""Host against device random draws at the refinement sample's sizes (lidiff_b200.rng): numpy's randn(1, 4 146 667, 3) and
torch's randperm(4 146 667) and randperm(1 036 666), each checked bit for bit against the host call; the share of logs resolved on
the host, the reservation rounds; then samples/s of the refinement train and validation samples (windows of 40 synthetic scans,
num_points 180 000, scripts/bench_refine_samples.py's sequence) with and without device_rng.  Prints one JSON line with the card
name, power limit and SM clock.

    python scripts/bench_device_rng.py [--reps 3] [--scans 40] [--samples 3] [--device cuda:0]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_eval import gpu_card                          # noqa: E402
from scripts.bench_refine_samples import NUM_POINTS, WINDOW, write_sequence  # noqa: E402

N_ROWS, N_GT = 4146667, 1036666


def clocks(index):
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception:
        return "unavailable"


def timed(fn, reps, sync):
    best = float("inf")
    for _ in range(reps):
        if sync:
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        if sync:
            torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return out, best * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scans", type=int, default=WINDOW)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args()
    from lidiff_b200 import rng
    from lidiff_b200.datasets_refine import TemporalKITTISet
    dev = torch.device(a.device)
    torch.cuda.set_device(dev)
    res = {"bench": "device_rng", "card": gpu_card(dev.index or 0), "clocks_sm_and_max": clocks(dev.index or 0)}
    rng.numpy_randn(1000, device=dev, random_state=np.random.RandomState(0))          # warm-up: module load, first launches
    rng.torch_randperm(1000, device=dev, generator=torch.Generator().manual_seed(0))

    st = {}
    rs_h, rs_d = np.random.RandomState(1), np.random.RandomState(1)
    ref, res["randn_host_ms"] = timed(lambda: rs_h.randn(1, N_ROWS, 3), a.reps, False)
    got, res["randn_device_ms"] = timed(lambda: rng.numpy_randn(1, N_ROWS, 3, device=dev, random_state=rs_d, stats=st), a.reps, True)
    assert np.array_equal(got.cpu().numpy().view(np.uint64), ref.view(np.uint64)), "randn differs from numpy"
    res["randn_deferred_fraction"] = round(st["deferred"] / st["pairs"], 5)
    res["randn_words"] = st["words"]
    for n, tag in ((N_ROWS, "randperm_4m"), (N_GT, "randperm_1m")):
        g_h, g_d = torch.Generator().manual_seed(2), torch.Generator().manual_seed(2)
        st = {}
        ref, res[f"{tag}_host_ms"] = timed(lambda: torch.randperm(n, generator=g_h), a.reps, False)
        got, res[f"{tag}_device_ms"] = timed(lambda: rng.torch_randperm(n, device=dev, generator=g_d, stats=st), a.reps, True)
        assert torch.equal(got.cpu(), ref), f"randperm({n}) differs from torch"
        res[f"{tag}_rounds"] = st["rounds"]
    for k in res:
        if k.endswith("_ms"):
            res[k] = round(res[k], 2)

    with tempfile.TemporaryDirectory() as root:
        write_sequence(os.path.join(root, "dataset", "sequences", "00"), a.scans)
        for split in ("validation", "train"):
            for device_rng in (False, True):
                ds = TemporalKITTISet(root, WINDOW, ["00"], split, 0.05, NUM_POINTS, "refine", device=dev, device_rng=device_rng)
                np.random.seed(0)
                torch.manual_seed(0)
                ds[0]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for k in range(a.samples):
                    ds[k % len(ds)]
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) / a.samples
                res[f"{split}_samples_per_s{'_device_rng' if device_rng else ''}"] = round(1 / dt, 3)
                del ds
    print(json.dumps(res))


if __name__ == "__main__":
    main()
