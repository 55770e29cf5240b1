#!/usr/bin/env python
"""Time of the scene-completion grid work (lidiff_b200.ssc) at the sizes eval_path meets: converting a sequence's worth of
synthetic grids (815, as many as sequence 08 has) to voxel centres, each GPU phase by CUDA events on device-resident chunks
(counting: three launches; emitting: one) and the whole ssc.grid_points call from host arrays by the host clock around work that
ends in a synchronise, against the numpy restatement of tests/ssc_reference.py per grid; voxelizing a 1.02 M-point cloud shaped
like a refined completion (numpy for comparison); and the confusion counts of one grid and of a chunk of grids.  Outputs are
checked bit for bit against the restatement in the same run, and the card, power limit and SM clock are read in it too.  Prints
one JSON line.

    python scripts/bench_ssc.py [--grids 815] [--density 0.05] [--reps 7] [--device cuda:0]
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
    ap.add_argument("--grids", type=int, default=815)
    ap.add_argument("--density", type=float, default=0.05)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    device = torch.device(args.device)
    torch.cuda.set_device(device)

    import ssc_reference as SR
    from lidiff_b200 import _lib
    from lidiff_b200 import ssc as S

    h = _lib.get_handle(device)
    g = np.random.default_rng(0)
    distinct = [SR.random_labels(g, args.density, 0.02) for _ in range(8)]
    seq = np.stack([distinct[i % 8] for i in range(args.grids)])                 # (G, N_VOXELS) uint16
    res = {"grids": args.grids, "density": args.density, "chunk": S.CHUNK, "gpu": gpu_state(device.index or 0)}

    # GPU phases on one device-resident chunk of labels
    chunk = torch.from_numpy(seq[:S.CHUNK]).view(torch.int16).to(device)
    off = torch.empty(S.CHUNK + 1, dtype=torch.int64, device=device)
    scratch = h.ssc_scratch(S.CHUNK)
    h.ssc_grid_count(chunk, _lib.SSC_LABELS, S.CHUNK, off, scratch)
    out = torch.empty((int(off[-1].item()), 3), dtype=torch.float64, device=device)
    res["chunk_points"] = out.shape[0]
    res["count_chunk_ms"] = _events(lambda: h.ssc_grid_count(chunk, _lib.SSC_LABELS, S.CHUNK, off, scratch), args.reps)
    res["emit_chunk_ms"] = _events(lambda: h.ssc_grid_points(S.CHUNK, off, scratch, out), args.reps)
    bits_chunk = torch.from_numpy(np.stack([SR.pack(SR.occupied(x)) for x in seq[:S.CHUNK]]).view(np.int32)).to(device)
    res["count_bits_chunk_ms"] = _events(lambda: h.ssc_grid_count(bits_chunk, _lib.SSC_BITS, S.CHUNK, off, scratch), args.reps)

    # the whole sequence from host arrays (upload, chunks, host reads, concatenation)
    res["grid_points_sequence_ms"] = _host(lambda: S.grid_points(seq, "labels", device=device), max(1, args.reps // 3))
    pts, offs = S.grid_points(seq, "labels", device=device)
    res["sequence_points"] = int(offs[-1])
    t0 = time.perf_counter()
    want = [SR.centres(SR.occupied(x)) for x in distinct]
    res["numpy_grid_points_per_grid_ms"] = (time.perf_counter() - t0) * 1e3 / len(distinct)
    got = pts.cpu().numpy()
    res["grid_points_bit_exact"] = bool(all(np.array_equal(got[offs[b]:offs[b + 1]], want[b % 8]) for b in range(args.grids)))
    del pts, got

    # voxelization of a refined-completion-sized cloud (1.02 M points within 50 m, half of them outside the SSC grid)
    cloud = np.concatenate([g.uniform([-50, -50, -3], [50, 50, 5], (1_020_000, 3))])
    cloud_d = torch.from_numpy(cloud).to(device)
    S.voxelize(cloud_d, device=device)
    res["voxelize_ms"] = _host(lambda: S.voxelize(cloud_d, device=device), args.reps)
    offsets = torch.tensor([0, cloud.shape[0]], dtype=torch.int64, device=device)
    vbits = torch.empty((1, S.N_WORDS), dtype=torch.int32, device=device)
    vinfo = torch.empty(16, dtype=torch.uint8, device=device)
    res["voxelize_kernel_ms"] = _events(lambda: h.ssc_voxelize(cloud_d, offsets, 1, vbits, vinfo), args.reps)
    t0 = time.perf_counter()
    want_bits, nf, outside = SR.voxelize(cloud)
    res["numpy_voxelize_ms"] = (time.perf_counter() - t0) * 1e3
    bits, dropped = S.voxelize(cloud_d, device=device)
    res["voxelize_bit_exact"] = bool(np.array_equal(bits.cpu().numpy().view(np.uint32), want_bits) and list(dropped) == [nf, outside])

    # confusion counts: one grid, and a chunk of grids, device-resident
    inv = torch.from_numpy(np.stack([SR.pack(g.random(S.N_VOXELS) < 0.05) for _ in range(S.CHUNK)]).view(np.int32)).to(device)
    conf = torch.empty((S.CHUNK, 3), dtype=torch.int64, device=device)
    res["confusion_one_grid_ms"] = _events(lambda: h.ssc_confusion(bits_chunk[:1], chunk[:1], inv[:1], 1, conf), args.reps)
    res["confusion_chunk_ms"] = _events(lambda: h.ssc_confusion(bits_chunk, chunk, inv, S.CHUNK, conf), args.reps)
    t0 = time.perf_counter()
    want_conf = SR.confusion(SR.pack(SR.occupied(seq[0])), seq[0], inv[0].cpu().numpy().view(np.uint32))
    res["numpy_confusion_one_grid_ms"] = (time.perf_counter() - t0) * 1e3
    h.ssc_confusion(bits_chunk[:1], chunk[:1], inv[:1], 1, conf)
    res["confusion_exact"] = tuple(conf[0].tolist()) == want_conf
    print(json.dumps(res))


if __name__ == "__main__":
    main()
