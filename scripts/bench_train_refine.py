#!/usr/bin/env python
"""One training step of the refinement network (lidiff_b200.tools.train_refine.train_step) at the reference's batch: 8 windows of
180 000 noisy points (num_points), 360 000 ground-truth points each, from seeded synthetic scans.  After --warmup untimed steps,
--steps timed steps report ms per step and its split by CUDA events: forward (TensorField -> offsets), loss (Chamfer forward), input
gradients (the forward convolution kernels on the adjoint maps), weight gradients (lb2_spconv_wgrad), the rest of backward (BN, ReLU,
Linear, Chamfer, gathers), and Adam.  Then, per weight-gradient shape (kvol, cin, cout, tensor stride) of the step, its kernel time
and achieved TFLOP/s, counting 2 cin cout FLOPs per present (input row, output row) pair, against the FP16x3 tensor-core roofline:
the data sheet's dense FP16 rate / 3 (three MMAs per product), in bench.py's roofline form.  Prints one JSON line with the card name
and power limit.

    python scripts/bench_train_refine.py [--steps 5] [--warmup 2] [--batch 8] [--points 180000] [--device cuda:0]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_eval import gpu_card                      # noqa: E402

PEAK_FP16_TFLOPS = 989.0          # H100 SXM data sheet, dense FP16 tensor (700 W card, not a measured ceiling)


def make_batch(b, n, seed=0):
    from lidiff_b200.synth import synthetic_scan
    full, noise = [], []
    for i in range(b):
        s = synthetic_scan(seed + i)
        g = np.random.default_rng(seed + i)
        s = s[np.linalg.norm(s, axis=1) < 50.0]
        full.append(s[g.choice(s.shape[0], 2 * n, replace=2 * n > s.shape[0])])
        noise.append(full[-1][:n] + np.clip(0.2 * g.standard_normal((n, 3)), -0.3, 0.3) * 0.1)
    return {"pcd_full": torch.from_numpy(np.stack(full)).float(), "pcd_noise": torch.from_numpy(np.stack(noise)).float()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--points", type=int, default=180000)
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args()
    dev = torch.device(a.device)
    torch.cuda.set_device(dev)
    from lidiff_b200 import me as ME
    from lidiff_b200 import metrics
    from lidiff_b200.minkunet import MinkUNet
    from lidiff_b200.tools import test_refine, train_refine

    cfg = {"data": {"resolution": 0.05}, "train": {"lr": 1e-4, "up_factor": 6}}
    torch.manual_seed(0)
    net = MinkUNet(in_channels=3, out_channels=18).to(dev).train()
    opt = train_refine.make_optimizer(net, cfg)
    batch = make_batch(a.batch, a.points)

    ev = defaultdict(list)                 # phase -> [(start, end)] of the current step
    shapes = defaultdict(list)             # (kvol, cin, cout, ts) -> [(start, end, pairs)]

    def timed(name, fn, key=None):
        def wrap(*args, **kw):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = fn(*args, **kw)
            e.record()
            ev[name].append((s, e))
            if key is not None:
                shapes[key(*args)].append((s, e))
            return r
        return wrap

    def wkey(layer, F, G, cm, ts):
        return (layer.kernel_volume, layer.in_channels, layer.out_channels, ts, "T" if layer.transposed else "")

    base = ME._ConvBase
    base._input_grad = timed("input_grad", base._input_grad)
    base._weight_grad = timed("weight_grad", base._weight_grad, key=wkey)
    orig_chamfer = test_refine.chamfer_distance
    test_refine.chamfer_distance = timed("loss", orig_chamfer)
    orig_net_forward = MinkUNet.forward
    MinkUNet.forward = timed("forward", orig_net_forward)

    def step():
        s, m, e = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        opt.zero_grad(set_to_none=True)
        s.record()
        _, loss = train_refine.refine_forward(net, batch, 0.05, 6, dev)
        loss.backward()
        m.record()
        opt.step()
        e.record()
        return s, m, e

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    ev.clear()
    shapes.clear()
    marks = [step() for _ in range(a.steps)]
    torch.cuda.synchronize()
    tot = lambda name: sum(s.elapsed_time(e) for s, e in ev[name]) / a.steps
    step_ms = sum(s.elapsed_time(e) for s, _, e in marks) / a.steps
    fb_ms = sum(s.elapsed_time(m) for s, m, _ in marks) / a.steps
    adam_ms = sum(m.elapsed_time(e) for _, m, e in marks) / a.steps
    fwd, loss_ms, dg, wg = tot("forward"), tot("loss"), tot("input_grad"), tot("weight_grad")

    # per-shape weight-gradient rate: present pairs from the maps of one more forward
    with torch.no_grad():
        xf = ME.utils.batched_coordinates(list(batch["pcd_noise"]), dtype=torch.float32, device=dev)
        field = ME.TensorField(features=xf[:, 1:], coordinates=torch.round(xf / 0.05), device=dev)
        net(field)
        cm = field.coordinate_manager
    peak = PEAK_FP16_TFLOPS / 3.0
    rows = []
    for (kvol, cin, cout, ts, t), lst in sorted(shapes.items()):
        ms = sum(s.elapsed_time(e) for s, e in lst) / len(lst)
        if kvol == 1:
            pairs = cm.level(ts).n
        elif kvol == 27:
            pairs = int((cm.kernel_map(ts, 3, 1, False) >= 0).sum().item())
        else:
            pairs = int((cm.kernel_map(ts, 2, 2, t == "T") >= 0).sum().item())
        tf = 2.0 * pairs * cin * cout / (ms * 1e-3) / 1e12
        rows.append({"kvol": kvol, "cin": cin, "cout": cout, "ts": ts, "transposed": t == "T", "calls_per_step": len(lst) // a.steps,
                     "pairs": pairs, "ms": round(ms, 3), "tflops": round(tf, 2), "share_of_roofline": round(tf / peak, 3)})
    best = max(rows, key=lambda r: r["ms"] * r["calls_per_step"])
    res = {"metric": "refine_train_step", "batch": a.batch, "points_per_window": a.points, "steps": a.steps,
           "level_rows": [cm.level(1 << l).n for l in range(5)],
           "step_ms": round(step_ms, 2),
           "split_ms": {"forward": round(fwd, 2), "loss": round(loss_ms, 2), "input_grad": round(dg, 2), "weight_grad": round(wg, 2),
                        "backward_rest": round(fb_ms - fwd - loss_ms - dg - wg, 2), "adam": round(adam_ms, 2)},
           "wgrad_shapes": rows,
           "roofline": {"kernel": f"k_spconv_wgrad {best['kvol']}:{best['cin']}->{best['cout']} ts{best['ts']}", "bound": "tensor",
                        "achieved": best["tflops"], "peak": round(peak, 1), "unit": "TFLOP/s",
                        "peak_src": "H100 SXM data sheet dense FP16 / 3 (FP16x3: three MMAs per product; not a measured ceiling)"},
           "gpu": gpu_card(dev.index or 0)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
