#!/usr/bin/env python
"""Time of open3d's uniform surface sampling (lidiff_b200.mesh) of 1 000 000 points from a 1000 x 1000-vertex height field
(1 996 002 triangles, tests/mesh_reference.height_field): each kernel of the call by CUDA events around single launches (the five
prepare kernels by torch.profiler in a separate pass, since lb2_mesh_sample_prepare launches them together), the MT19937 words and
the sampling kernel, the whole sample_points_uniformly call and the public Metrics3D.convert_to_pcd of a shim TriangleMesh (host
clock around work that ends in a synchronise, host copies included), and the numpy restatement of tests/mesh_reference.py on the
host with a bit-exactness check, with the card, power limit and SM clock read in the same run.  Prints one JSON line.

    python scripts/bench_mesh_sample.py [--reps 7] [--side 1000] [--points 1000000] [--device cuda:0]
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


def _events(fn, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def _host(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--side", type=int, default=1000)
    ap.add_argument("--points", type=int, default=1000000)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    device = torch.device(args.device)
    torch.cuda.set_device(device)
    from torch.profiler import ProfilerActivity, profile

    import mesh_reference as MR
    from lidiff_b200 import _lib
    from lidiff_b200 import mesh as MESH
    from lidiff_b200 import metrics as M
    from lidiff_b200.rng import _words
    from lidiff_b200.shims.open3d import geometry, utility

    v, t = MR.height_field(args.side, seed=7, offset=1e5)
    n = args.points
    h = _lib.get_handle(device)
    vv, tt = MESH._mesh(v, t, h.device)
    key, pos = MESH.seed_state(1)
    area = torch.empty(t.shape[0], dtype=torch.float64, device=device)
    info = torch.empty(24, dtype=torch.uint8, device=device)
    scratch = h.mesh_sample_scratch(t.shape[0])
    out = torch.empty((n, 3), dtype=torch.float64, device=device)
    holder = {}

    def prepare():
        h.mesh_sample_prepare(vv, tt, n, area, info, scratch)

    def words():
        holder["w"] = _words(h, key, pos, 4 * n)[0]

    def sample():
        h.mesh_sample_points(vv, tt, scratch, holder["w"], n, out)

    for f in (prepare, words, sample):                            # warm-up
        f()
    torch.cuda.synchronize()
    res = {"triangles": int(t.shape[0]), "points": n, "gpu": gpu_state(device.index or 0)}
    res["prepare_ms"] = _events(prepare, args.reps)
    res["mt19937_words_ms"] = _events(words, args.reps)
    res["sample_ms"] = _events(sample, args.reps)

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            prepare()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if "k_mesh" in e.key:
            per[e.key.split("(")[0]] = round(e.device_time_total / 1e3 / e.count, 4)     # ms per launch
    res["prepare_kernels_ms"] = per

    res["sample_points_uniformly_ms"] = _host(lambda: MESH.sample_points_uniformly(v, t, n, key, pos, device=device), args.reps)
    mesh = geometry.TriangleMesh(v, t)
    utility.random.seed(1)
    res["convert_to_pcd_ms"] = _host(lambda: M.Metrics3D.convert_to_pcd(mesh), args.reps)

    got = MESH.sample_points_uniformly(v, t, n, key, pos, device=device)[0].cpu().numpy()
    t0 = time.perf_counter()
    want = MR.sample_stream(v, t, n, key, pos)[0]
    res["numpy_restatement_ms"] = (time.perf_counter() - t0) * 1e3
    res["bit_exact"] = bool(np.array_equal(got.view(np.uint64), want.view(np.uint64)))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
