#!/usr/bin/env python
"""One training step of the diffusion network (lidiff_b200.tools.train_diffusion.train_step) at the config's batch: 2 scans of
180 000 ground-truth points and 18 000 part points each, from seeded synthetic scans.  The conditional and the unconditional step
are timed separately (the switch is forced): after --warmup untimed steps of each, --steps timed steps report ms per step and its
split by CUDA events: forward, gate backward (GateMul: lb2_gate_mul + lb2_segment_dot, with the sort that orders the rows), input
gradients, weight gradients (lb2_spconv_wgrad), the rest of backward (BN, ReLU, the MLPs on part rows, gathers), and Adam.

Then, on the step's own gate indices (every gate's idx, widths and rows), lb2_segment_dot(G, X) against what it replaces:
rowsum.index_sum of the materialised product G * X (lb2_segment_sum, one warp per segment) on the same order and offsets, both
without the sort.  Prints one JSON line with the card name, power limit and clocks as read.

    python scripts/bench_train_diffusion.py [--steps 5] [--warmup 2] [--batch 2] [--points 180000] [--device cuda:0]
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


def make_batch(b, n, seed=0):
    from lidiff_b200.synth import synthetic_scan
    full, part = [], []
    for i in range(b):
        s = synthetic_scan(seed + i)
        g = np.random.default_rng(seed + i)
        s = s[np.linalg.norm(s, axis=1) < 50.0]
        full.append(s[g.choice(s.shape[0], n, replace=n > s.shape[0])])
        part.append(full[-1][g.choice(n, n // 10, replace=False)])
    return {"pcd_full": torch.from_numpy(np.stack(full)).float(), "pcd_part": torch.from_numpy(np.stack(part)).float()}


def gpu_clocks(index):
    """SM clock now and its maximum as nvidia-smi reports them, or that they could not be read"""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        now, top = [c.strip() for c in r.stdout.strip().split(",")[:2]]
        return {"sm_clock": now, "sm_clock_max": top}
    except Exception:
        return {"sm_clock": "unavailable", "sm_clock_max": "unavailable"}


def event_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--points", type=int, default=180000)
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args()
    dev = torch.device(a.device)
    torch.cuda.set_device(dev)
    from lidiff_b200 import _lib, gate
    from lidiff_b200 import me as ME
    from lidiff_b200.tools import train_diffusion as T

    cfg = {"data": {"resolution": 0.05}, "train": {"lr": 1e-4, "uncond_prob": 0.1},
           "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "reg_weight": 5.0},
           "model": {"out_dim": 96}}
    somac = T.sqrt_one_minus_alphas_cumprod(cfg)
    torch.manual_seed(0)
    nets = T.DiffusionNets(cfg).to(dev).train()
    opt, _ = T.make_optimizer(nets, cfg)
    batch = make_batch(a.batch, a.points)

    ev = defaultdict(list)
    gates = []                                # (G, x, idx32, table rows) of the last step's gate backwards

    def timed(name, fn, keep=None):
        def wrap(*args, **kw):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = fn(*args, **kw)
            e.record()
            ev[name].append((s, e))
            if keep is not None:
                keep(*args)
            return r
        return wrap

    def keep_gate(ctx, G):
        x, table, idx32 = ctx.saved_tensors
        gates.append((G.detach().contiguous(), x.detach(), idx32, table.shape[0]))

    ME._ConvBase._input_grad = timed("input_grad", ME._ConvBase._input_grad)
    ME._ConvBase._weight_grad = timed("weight_grad", ME._ConvBase._weight_grad)
    gate.GateMul.backward = staticmethod(timed("gate_backward", gate.GateMul.backward, keep=keep_gate))
    T.DiffusionNets.forward = timed("forward", T.DiffusionNets.forward)

    def step():
        s, m, e = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        opt.zero_grad(set_to_none=True)
        s.record()
        T.training_forward(nets, batch, cfg, somac, dev)["loss"].backward()
        m.record()
        opt.step()
        e.record()
        return s, m, e

    res = {"metric": "diffusion_train_step", "batch": a.batch, "points_per_scan": a.points, "steps": a.steps}
    h = _lib.get_handle(dev)
    for mode, prob in (("conditional", -1.0), ("unconditional", 2.0)):
        cfg["train"]["uncond_prob"] = prob
        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        ev.clear()
        gates.clear()
        marks = [step() for _ in range(a.steps)]
        torch.cuda.synchronize()
        tot = lambda name: sum(s.elapsed_time(e) for s, e in ev[name]) / a.steps   # noqa: E731
        fb = sum(s.elapsed_time(m) for s, m, _ in marks) / a.steps
        fwd, gb, dg, wg = tot("forward"), tot("gate_backward"), tot("input_grad"), tot("weight_grad")
        out = {"step_ms": round(sum(s.elapsed_time(e) for s, _, e in marks) / a.steps, 2),
               "split_ms": {"forward": round(fwd, 2), "gate_backward": round(gb, 2), "input_grad": round(dg, 2), "weight_grad": round(wg, 2),
                            "backward_rest": round(fb - fwd - gb - dg - wg, 2),
                            "adam": round(sum(m.elapsed_time(e) for _, m, e in marks) / a.steps, 2)},
               "peak_memory_gib": round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2)}
        rows = []
        for G, x, idx32, n in gates[-8:]:                       # the last step's eight gates, in backward order (up4 first)
            idx = idx32.long()
            order = torch.sort(idx, stable=True).indices
            offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
            torch.cumsum(torch.bincount(idx, minlength=n), 0, out=offsets[1:])
            o1, o2 = torch.empty(n, x.shape[1], device=dev), torch.empty(n, x.shape[1], device=dev)
            dot_ms = event_ms(lambda: h.segment_dot(G, x, order, offsets, o1), 20)
            prod = G * x
            mul_ms = event_ms(lambda: torch.mul(G, x, out=prod), 20)
            sum_ms = event_ms(lambda: h.segment_sum(prod, order, offsets, o2), 3)
            rows.append({"rows": x.shape[0], "c": x.shape[1], "segments": n, "longest": int((offsets[1:] - offsets[:-1]).max()),
                         "segment_dot_ms": round(dot_ms, 4), "product_ms": round(mul_ms, 4), "segment_sum_ms": round(sum_ms, 3),
                         "gb_per_s": round(2 * x.numel() * 4 / dot_ms / 1e6, 1),
                         "max_rel_diff": float(((o1 - o2).abs().max() / o2.abs().max().clamp_min(1e-30)).item())})
        out["gates"] = rows
        out["segment_dot_ms_all_gates"] = round(sum(r["segment_dot_ms"] for r in rows), 3)
        out["product_plus_segment_sum_ms_all_gates"] = round(sum(r["product_ms"] + r["segment_sum_ms"] for r in rows), 2)
        res[mode] = out
    res["gpu"] = {**gpu_card(dev.index or 0), **gpu_clocks(dev.index or 0)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
