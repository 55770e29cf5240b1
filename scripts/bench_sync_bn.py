#!/usr/bin/env python
"""The synchronised batch norm's kernels (lb2_sync_bn_*, called directly, without collectives) against nn.BatchNorm1d's training
forward + backward on the same tensors, for every BN input of a conditional diffusion training step (2 x 180 000 points) and of a
refinement training step (8 x 180 000 points): the shapes are recorded from one forward of each network on seeded synthetic scans.
Per shape: CUDA-event ms of the seven sync-BN calls (forward + backward) and of BatchNorm1d forward + backward, and the sync path's
bytes (x read 4 times and y written in the forward; dy and x read 3 times and dx written in the backward) over its time against
3.35 TB/s.  Then the ms per step of a 2-rank diffusion training step with both ranks on one GPU over gloo (a functional figure: two
processes share the device) and, with two or more GPUs visible, weak scaling: ms per step at W = 1, 2, 4, 8 ranks over NCCL, one
GPU and 2 x 180 000 points per rank.  Prints one JSON line with the card name and power limit as read.

    python scripts/bench_sync_bn.py [--reps 20] [--ddp-steps 3] [--device cuda:0]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_eval import gpu_card                      # noqa: E402
from scripts.bench_train_diffusion import event_ms, make_batch  # noqa: E402

HBM = 3.35e12


def bn_shapes(which, dev):
    """(rows, channels) of every BN input of one training forward"""
    from lidiff_b200 import me as ME
    shapes = []
    hook = lambda m, inp, out: shapes.append(tuple(inp[0].F.shape))  # noqa: E731
    if which == "diffusion":
        from lidiff_b200.tools import train_diffusion as T
        cfg = {"data": {"resolution": 0.05}, "train": {"uncond_prob": 0.0}, "diff": {"t_steps": 1000, "reg_weight": 5.0,
               "beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear"}, "model": {"out_dim": 96}}
        net = T.DiffusionNets(cfg).to(dev)
        batch = make_batch(2, 180_000)
        run = lambda: T.training_forward(net, batch, cfg, T.sqrt_one_minus_alphas_cumprod(cfg), dev)  # noqa: E731
    else:
        from lidiff_b200.minkunet import MinkUNet
        from lidiff_b200.tools.test_refine import refine_batch
        net = MinkUNet(in_channels=3, out_channels=18).to(dev)
        full = make_batch(8, 180_000)["pcd_full"]
        run = lambda: refine_batch.__wrapped__(net, {"pcd_noise": full, "pcd_full": full}, 0.05, 6, dev)  # noqa: E731
    hs = [m.register_forward_hook(hook) for m in net.modules() if isinstance(m, ME.MinkowskiBatchNorm)]
    with torch.no_grad():
        run()
    for h in hs:
        h.remove()
    return shapes


def time_shape(n, c, dev, reps):
    from lidiff_b200 import _lib
    h = _lib.get_handle(dev)
    g = torch.Generator(device=dev).manual_seed(n + c)
    x = torch.randn(n, c, device=dev, generator=g)
    dy = torch.randn(n, c, device=dev, generator=g)
    i64 = dict(dtype=torch.int64, device=dev)
    mw, sw, qw, bmw, bsw = (torch.empty(k * c + e, **i64) for k, e in ((2, 0), (2, 1), (4, 0), (3, 0), (4, 0)))
    mean, var, invstd = (torch.empty(c, dtype=torch.float64, device=dev) for _ in range(3))
    gamma, beta = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    y, dx = torch.empty_like(x), torch.empty_like(x)
    dg, db = torch.empty(c, device=dev), torch.empty(c, device=dev)

    def sync():
        h.sync_bn_max(x, mw)
        h.sync_bn_sum(x, mw, sw)
        h.sync_bn_sumsq(x, mw, sw, mean, qw)
        h.sync_bn_apply(x, mw, sw, mean, qw, gamma, beta, 1e-5, 0.1, rm, rv, var, invstd, y)
        h.sync_bn_backward_max(dy, x, mean, invstd, bmw)
        h.sync_bn_backward_sum(dy, x, mean, invstd, bmw, bsw, dg, db)
        h.sync_bn_backward_apply(dy, x, mean, invstd, gamma, bmw, bsw, sw[2 * c:], dx)

    bn = torch.nn.BatchNorm1d(c).to(dev).train()
    xr = x.clone().requires_grad_(True)

    def torch_bn():
        xr.grad = None
        bn(xr).backward(dy)

    t_sync, t_bn = event_ms(sync, reps), event_ms(torch_bn, reps)
    nbytes = 12 * n * c * 4
    return {"rows": n, "c": c, "sync_ms": round(t_sync, 4), "bn1d_ms": round(t_bn, 4),
            "sync_GBps": round(nbytes / (t_sync * 1e-3) / 1e9, 1), "sync_share_of_hbm": round(nbytes / (t_sync * 1e-3) / HBM, 3)}


def _ddp_rank(rank, world, tmp, steps, backend):
    """a diffusion training step at 2 x 180 000 points per rank, wrapped as the CLIs wrap it: ms per step (rank 0 writes it).
    gloo: every rank on cuda:0; nccl: rank r on cuda:r.  world 1: no process group (the single-process step)."""
    import torch.distributed as dist
    from lidiff_b200 import ddp
    from lidiff_b200.tools import train_diffusion as T
    dev = torch.device("cuda", 0 if backend == "gloo" else rank)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group(backend, init_method=f"file://{os.path.join(tmp, 'rdv')}", rank=rank, world_size=world)
    cfg = {"data": {"resolution": 0.05}, "train": {"uncond_prob": 0.0, "lr": 1e-4}, "diff": {"t_steps": 1000, "reg_weight": 5.0,
           "beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear"}, "model": {"out_dim": 96}}
    nets = T.DiffusionNets(cfg).to(dev)
    opt, _ = T.make_optimizer(nets, cfg)
    model, nets = ddp.wrap(nets, ddp.Run(rank, world, dev))
    model.train()
    somac = T.sqrt_one_minus_alphas_cumprod(cfg)
    batch = make_batch(2, 180_000, seed=10 * rank)
    T.train_step(model, opt, batch, cfg, somac, dev)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    for _ in range(steps):
        T.train_step(model, opt, batch, cfg, somac, dev)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    if rank == 0:
        with open(os.path.join(tmp, "ms"), "w") as f:
            f.write(str((time.perf_counter() - t0) * 1e3 / steps))
    if world > 1:
        dist.destroy_process_group()


def ddp_ms(world, steps, backend):
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as tmp:
        mp.start_processes(_ddp_rank, args=(world, tmp, steps, backend), nprocs=world, start_method="spawn")
        return round(float(open(os.path.join(tmp, "ms")).read()), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ddp-steps", type=int, default=3)
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args()
    dev = torch.device(a.device)
    res = {**gpu_card(dev.index or 0)}
    for which in ("diffusion", "refine"):
        rows = [time_shape(n, c, dev, a.reps) for n, c in bn_shapes(which, dev)]
        res[which] = {"bn_layers": len(rows), "sync_ms_total": round(sum(r["sync_ms"] for r in rows), 3),
                      "bn1d_ms_total": round(sum(r["bn1d_ms"] for r in rows), 3), "layers": rows}
        torch.cuda.empty_cache()
    if a.ddp_steps > 0:
        res["ddp_2rank_one_gpu_gloo_ms_per_step"] = ddp_ms(2, a.ddp_steps, "gloo")
        # weak scaling: W ranks over NCCL, one GPU each, 2 x 180 000 points per rank
        ngpu = torch.cuda.device_count()
        if ngpu < 2:
            res["multi_gpu_weak_scaling"] = "not measured (one GPU visible)"
        else:
            ws = [w for w in (1, 2, 4, 8) if w <= ngpu]
            res["multi_gpu_weak_scaling_ms_per_step"] = {str(w): ddp_ms(w, a.ddp_steps, "nccl") for w in ws}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
