"""Rank bodies for the multi-process synchronised batch-norm tests (run by fake_sync_bn_backend.run_ranks, importable by name)."""
import numpy as np
import torch


def bn_rank(rank, world, x_parts, g_parts, gamma, beta, device):
    """one MinkowskiSyncBatchNorm forward + backward on this rank's rows: y, dx, the local and the DDP-averaged parameter gradients,
    mean / var / invstd as saved, and the running statistics"""
    import torch.distributed as dist
    from lidiff_b200 import me as ME
    if device != "cpu":
        torch.cuda.set_device(0)
    c = x_parts[rank].shape[1]
    layer = ME.MinkowskiSyncBatchNorm.convert_sync_batchnorm(ME.MinkowskiBatchNorm(c)).to(device)
    with torch.no_grad():
        layer.bn.weight.copy_(torch.from_numpy(gamma))
        layer.bn.bias.copy_(torch.from_numpy(beta))
    layer.train()
    x = torch.from_numpy(x_parts[rank]).to(device).requires_grad_(True)
    st = ME.SparseTensor(x, coordinate_manager=object())
    saved = {}
    h = ME._lib.get_handle(x.device)
    orig = h.sync_bn_apply

    def spy(*a):                        # mean, var and invstd as the layer computed them (arguments 3, 11 and 12)
        orig(*a)
        saved["mean"], saved["var"], saved["invstd"] = (a[i].cpu().numpy().copy() for i in (3, 11, 12))

    h.sync_bn_apply = spy
    try:
        y = layer(st).F
    finally:
        del h.sync_bn_apply
    (y * torch.from_numpy(g_parts[rank]).to(device)).sum().backward()
    dg, db = layer.bn.weight.grad.clone(), layer.bn.bias.grad.clone()
    avg = torch.cat([dg, db])
    dist.all_reduce(avg)
    avg /= world
    return {"y": y.detach().cpu().numpy(), "dx": x.grad.cpu().numpy(), "dgamma": dg.cpu().numpy(), "dbeta": db.cpu().numpy(),
            "avg_dgamma": avg[:c].cpu().numpy(), "avg_dbeta": avg[c:].cpu().numpy(), **saved,
            "running_mean": layer.bn.running_mean.cpu().numpy(), "running_var": layer.bn.running_var.cpu().numpy(),
            "num_batches_tracked": int(layer.bn.num_batches_tracked)}


def rows_of(parts, perm, n):
    """the ranks' row blocks put back in the original row order"""
    out = np.empty((n,) + parts[0].shape[1:], dtype=parts[0].dtype)
    out[perm] = np.concatenate(parts)
    return out


def _diffusion_cfg():
    return {"experiment": {"id": "D"}, "data": {"resolution": 0.05, "num_points": 300},
            "train": {"lr": 1e-3, "uncond_prob": 0.1, "uncond_w": 6.0, "max_epoch": 1, "batch_size": 2},
            "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 2, "reg_weight": 5.0},
            "model": {"out_dim": 96}}


def _rank_batch(which, rank, n):
    """the first batch of `rank` in train_rank: (diffusion) pcd_full / pcd_part, (refine) pcd_noise / pcd_full"""
    g = torch.Generator().manual_seed(100 + rank)
    if which == "diffusion":
        full = torch.randn(2, n, 3, generator=g) * torch.tensor([2.0, 2.0, 0.4])
        return g, {"pcd_full": full, "pcd_part": full[:, : n // 3].clone()}
    full = torch.randn(2, 6 * n, 3, generator=g) * torch.tensor([2.0, 2.0, 0.4])
    return g, {"pcd_noise": full[:, :n] + 0.01 * torch.randn(2, n, 3, generator=g), "pcd_full": full}


def _make_net(which, dev):
    """(net, optimizer, cfg, somac) as the CLIs build them, after set_deterministic()"""
    if which == "diffusion":
        from lidiff_b200.tools import train_diffusion as T
        cfg = _diffusion_cfg()
        net = T.DiffusionNets(cfg).to(dev)
        return net, T.make_optimizer(net, cfg)[0], cfg, T.sqrt_one_minus_alphas_cumprod(cfg)
    from lidiff_b200.minkunet import MinkUNet
    from lidiff_b200.tools import train_refine as T
    cfg = {"data": {"resolution": 0.05}, "train": {"lr": 1e-3, "up_factor": 6}}
    net = MinkUNet(in_channels=3, out_channels=18).to(dev)
    return net, T.make_optimizer(net, cfg), cfg, None


def _running_stats(net):
    return {k: v.detach().cpu().clone() for k, v in net.state_dict().items() if k.endswith(("running_mean", "running_var"))}


def train_rank(rank, world, which, n, device, steps=2):
    """`steps` data-parallel training steps of one network (sync BN + DDP, as the CLIs wrap it) on rank-specific batches of n points
    per cloud: every parameter after the steps (flattened, in parameter order), the (DDP-averaged) parameter gradients and the BN
    running statistics of the first step, and how many BN layers of the wrapped model are synchronised / plain"""
    from lidiff_b200 import ddp
    from lidiff_b200 import me as ME
    from lidiff_b200.tools import train_diffusion as TD
    from lidiff_b200.tools import train_refine as TR
    from lidiff_b200.tools.test_completion import set_deterministic
    if device != "cpu":
        torch.cuda.set_device(0)
    set_deterministic()
    dev = torch.device(device if device == "cpu" else "cuda:0")
    run = ddp.Run(rank, world, dev)
    net, opt, cfg, somac = _make_net(which, dev)
    model, net = ddp.wrap(net, run)
    g, first = _rank_batch(which, rank, n)
    bns = [m for m in model.modules() if isinstance(m, ME.MinkowskiBatchNorm)]

    def step(batch):
        if which == "diffusion":
            return TD.train_step(model, opt, batch, cfg, somac, dev)
        return TR.train_step(model, opt, batch, cfg, dev)

    model.train()
    grads = stats = None
    for k in range(steps):
        step(first if k == 0 else _next_batch(which, g, n))
        if k == 0:
            grads = [p.grad.detach().cpu().double().clone() for p in net.parameters()]
            stats = _running_stats(net)
    params = torch.cat([p.detach().cpu().reshape(-1) for p in net.parameters()]).numpy()
    return {"params": params, "grads": grads, "running": stats, "state_keys": list(net.state_dict().keys()),
            "sync_bns": sum(isinstance(m, ME.MinkowskiSyncBatchNorm) for m in bns),
            "plain_bns": sum(not isinstance(m, ME.MinkowskiSyncBatchNorm) for m in bns)}


def _next_batch(which, g, n):
    if which == "diffusion":
        full = torch.randn(2, n, 3, generator=g) * torch.tensor([2.0, 2.0, 0.4])
        return {"pcd_full": full, "pcd_part": full[:, : n // 3].clone()}
    full = torch.randn(2, 6 * n, 3, generator=g) * torch.tensor([2.0, 2.0, 0.4])
    return {"pcd_noise": full[:, :n] + 0.01 * torch.randn(2, n, 3, generator=g), "pcd_full": full}


def union_first_step(which, n, world, device):
    """what train_rank's first step should compute, in one process without synchronised batch norm or DDP: the gradients of
    (1 / W) sum_r loss_r with batch statistics over the union of the ranks' rows (one forward over every rank's clouds), and the BN
    running statistics after it.  The ranks draw training_forward's random numbers from the same seeds (set_deterministic), so
    every rank's noise, time steps and unconditional switch are the draws replayed here once."""
    from lidiff_b200.tools import train_diffusion as TD
    from lidiff_b200.tools import train_refine as TR
    from lidiff_b200.tools.test_completion import set_deterministic
    set_deterministic()
    dev = torch.device(device if device == "cpu" else "cuda:0")
    net, _, cfg, somac = _make_net(which, dev)
    net.train()
    batches = [_rank_batch(which, r, n)[1] for r in range(world)]
    union = {k: torch.cat([b[k] for b in batches]) for k in batches[0]}
    if which == "refine":
        # pytorch3d's Chamfer loss is the mean over clouds: over the union it is the mean of the ranks' losses
        TR.refine_forward(net, union, cfg["data"]["resolution"], cfg["train"]["up_factor"], dev)[1].backward()
    else:
        full0 = batches[0]["pcd_full"]
        noise = torch.randn(full0.shape, device=dev)
        t = torch.randint(0, cfg["diff"]["t_steps"], size=(full0.shape[0],))
        uncond = not (torch.rand(1) > cfg["train"]["uncond_prob"] or full0.shape[0] == 1)
        samples = torch.cat([b["pcd_full"].to(dev) + somac[t][:, None, None].to(dev) * noise for b in batches])
        part = union["pcd_part"].to(dev)
        x_full = TD.points_to_tensor(samples, cfg["data"]["resolution"], dev)
        x_part = TD.points_to_tensor(torch.zeros_like(part) if uncond else part, cfg["data"]["resolution"], dev)
        out = net(x_full, x_part, t.repeat(world).to(dev))
        loss = 0.0
        for r in range(world):
            d = out[2 * r: 2 * r + 2]
            loss = loss + torch.nn.functional.mse_loss(d, noise) + cfg["diff"]["reg_weight"] * (d.mean() ** 2 + (d.std() - 1.0) ** 2)
        (loss / world).backward()
    return {"grads": [p.grad.detach().cpu().double().clone() for p in net.parameters()], "running": _running_stats(net)}
