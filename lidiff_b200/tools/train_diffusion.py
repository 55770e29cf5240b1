"""Train the diffusion network on SemanticKITTI — single-process counterpart of the reference's
`python train.py -c config.yaml [-w W] [-ckpt C]` (lidiff/train.py, DiffusionPoints.training_step / validation_step /
configure_optimizers, lidiff/models/models.py:180-217, 219-262, 337-346).

Every step draws training_step's random numbers in its order (the noise on the device, the time steps and the unconditional switch
from torch's host generator), noises `pcd_full` towards step t of the linear schedule, voxelises it at the config's resolution, runs
MinkGlobalEnc on the part cloud (or on one voxel at the origin per scan when the switch says unconditional) and MinkUNetDiff on the
noisy cloud, and takes one Adam step (lr = train.lr, betas (0.9, 0.999)) on loss_mse + reg_weight (loss_mean + loss_std).
ExponentialLR(0.5) steps once every 5 epochs.  Every 5 epochs the first validation batch is completed from its partial scan tiled
10 times with the current weights (DiffCompletion, diff.s_steps denoising steps) and scored after the completion's range and height
filter, as tools/test_completion scores it: Chamfer mean / std, precision / recall / F-score.  After every epoch
<out>/<experiment.id>_epoch=NN.ckpt holds the Lightning checkpoint fields the reference, tools/test_completion and DiffCompletion read:
state_dict (partial_enc.*, model.*), optimizer_states, lr_schedulers, epoch, global_step, hyper_parameters.

--max-steps N (not in the reference) stops this run after N optimiser steps and writes the checkpoint of the epoch it stopped in.

Under torchrun every rank trains on its own shard (lidiff_b200.ddp): synchronised batch norm, DistributedDataParallel averaging the
gradients, no learning-rate scaling, `train.n_gpus` = the world size in hyper_parameters.  Rank 0 prints the mean over ranks of the
logged scalars and of the validation scores (each rank completes the first batch of its own validation shard) and writes the
checkpoint, which loads unchanged in a single process.  TensorBoard and the open3d viewer are not built.

    python -m lidiff_b200.tools.train_diffusion -c lidiff/config/config.yaml
    torchrun --nproc-per-node 8 -m lidiff_b200.tools.train_diffusion -c lidiff/config/config.yaml
    python -m lidiff_b200.tools.train_diffusion -c config.yaml -ckpt experiments/prob10_5p0reg/checkpoints/prob10_5p0reg_epoch=04.ckpt
"""
from __future__ import annotations

import os

import click
import numpy as np
import torch
import torch.nn as nn
import yaml

from .. import ddp
from .. import me as ME
from ..datasets import TemporalKittiDataModule
from ..minkunet import MinkGlobalEnc, MinkUNetDiff
from .test_completion import set_deterministic

VAL_EVERY = 5
LR_EVERY = 5
LOGGED = ("loss_mse", "loss_mean", "loss_std", "loss", "var", "std")


class DiffusionNets(nn.Module):
    """the two trained networks under DiffusionPoints' attribute names, so that state_dict() has its keys"""

    def __init__(self, cfg):
        super().__init__()
        self.partial_enc = MinkGlobalEnc(in_channels=3, out_channels=cfg["model"]["out_dim"])
        self.model = MinkUNetDiff(in_channels=3, out_channels=cfg["model"]["out_dim"])

    def forward(self, x_full, x_part, t):
        return self.model(x_full, x_full.sparse(), self.partial_enc(x_part), t).reshape(t.shape[0], -1, 3)


def sqrt_one_minus_alphas_cumprod(cfg) -> torch.Tensor:
    """(t_steps,) fp32 on the host, as DiffusionPoints.__init__ computes it (models.py:24-49)"""
    d = cfg["diff"]
    if d["beta_func"] != "linear":
        raise ValueError(f"diff.beta_func '{d['beta_func']}' is not implemented: only the 'linear' schedule is")
    betas = torch.linspace(d["beta_start"], d["beta_end"], d["t_steps"])
    acp = torch.tensor(np.cumprod((1.0 - betas).numpy(), axis=0), dtype=torch.float32)
    return torch.sqrt(1.0 - acp)


def points_to_tensor(points, resolution, device):
    """models.py:162-178: features the float32 points, coordinates [b, round(x / resolution)] (feats_to_coord uses neither mean nor std)"""
    feats = ME.utils.batched_coordinates(list(points[:]), dtype=torch.float32, device=device)
    coords = feats.clone()
    coords[:, 1:] = torch.round(feats[:, 1:] / resolution)
    return ME.TensorField(features=feats[:, 1:], coordinates=coords, quantization_mode=ME.SparseTensorQuantizationMode.UNWEIGHTED_AVERAGE,
                          minkowski_algorithm=ME.MinkowskiAlgorithm.SPEED_OPTIMIZED, device=device)


def training_forward(nets, batch, cfg, somac, device) -> dict:
    """training_step (models.py:180-217): the logged scalars as tensors, 'loss' with its graph, and 'uncond' (bool)"""
    full = batch["pcd_full"].to(device)
    noise = torch.randn(full.shape, device=device)
    t = torch.randint(0, cfg["diff"]["t_steps"], size=(full.shape[0],))
    t_sample = full + somac[t][:, None, None].to(device) * noise
    resolution = cfg["data"]["resolution"]
    x_full = points_to_tensor(t_sample, resolution, device)
    uncond = not (torch.rand(1) > cfg["train"]["uncond_prob"] or full.shape[0] == 1)
    part = batch["pcd_part"].to(device)
    x_part = points_to_tensor(torch.zeros_like(part) if uncond else part, resolution, device)
    denoise_t = nets(x_full, x_part, t.to(device))
    loss_mse = nn.functional.mse_loss(denoise_t, noise)
    loss_mean = denoise_t.mean() ** 2
    loss_std = (denoise_t.std() - 1.0) ** 2
    sq = (denoise_t.detach() - noise) ** 2
    return {"loss_mse": loss_mse.detach(), "loss_mean": loss_mean.detach(), "loss_std": loss_std.detach(),
            "loss": loss_mse + cfg["diff"]["reg_weight"] * (loss_mean + loss_std), "var": sq.var(), "std": sq.std(), "uncond": uncond}


def make_optimizer(nets, cfg):
    """configure_optimizers (models.py:337-346): (Adam, ExponentialLR(0.5) to be stepped every LR_EVERY epochs)"""
    opt = torch.optim.Adam(nets.parameters(), lr=float(cfg["train"]["lr"]), betas=(0.9, 0.999))
    return opt, torch.optim.lr_scheduler.ExponentialLR(opt, 0.5)


def train_step(nets, opt, batch, cfg, somac, device) -> dict:
    """one training_step + optimizer step; returns the logged scalars (detached)"""
    opt.zero_grad(set_to_none=True)
    out = training_forward(nets, batch, cfg, somac, device)
    out["loss"].backward()
    opt.step()
    out["loss"] = out["loss"].detach()
    return out


def end_epoch(sched, epoch: int):
    if (epoch + 1) % LR_EVERY == 0:
        sched.step()


def validate(nets, batch, cfg, device):
    """validation_step on one batch (models.py:219-262): (cd_mean, cd_std, precision, recall, fscore)"""
    from ..metrics import ChamferDistance, PrecisionRecall
    from ..pipeline import DiffCompletion
    sd_enc = {k: v.detach().clone() for k, v in nets.partial_enc.state_dict().items()}
    sd_diff = {k: v.detach().clone() for k, v in nets.model.state_dict().items()}
    pipe = DiffCompletion(state_dicts={"enc": sd_enc, "diff": sd_diff}, denoising_steps=int(cfg["diff"]["s_steps"]),
                          cond_weight=cfg["train"]["uncond_w"], device=device,
                          hparams={"data": {"resolution": cfg["data"]["resolution"], "num_points": cfg["data"]["num_points"]},
                                   "diff": {k: cfg["diff"][k] for k in ("beta_start", "beta_end", "t_steps")}})
    resolution = cfg["data"]["resolution"]
    chamfer, prec_rec = ChamferDistance(), PrecisionRecall(resolution, 2 * resolution, 100)
    for i, (_, post) in enumerate(pipe.complete_scans(batch["pcd_part"].repeat(1, 10, 1), preprocessed=True, fresh=True)):
        gt = batch["pcd_full"][i].double()
        chamfer.update(gt, post)
        prec_rec.update(gt, post)
    del pipe                            # the engine's buffers go back to the device before the next training step
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    return (*chamfer.compute(), *prec_rec.compute_auc())


def checkpoint_path(out: str, cfg, epoch: int) -> str:
    return os.path.join(out, f"{cfg['experiment']['id']}_epoch={epoch:02d}.ckpt")


def save_checkpoint(path, nets, opt, sched, cfg, epoch: int, global_step: int):
    torch.save({"state_dict": {k: v.detach().cpu() for k, v in nets.state_dict().items()}, "optimizer_states": [opt.state_dict()],
                "lr_schedulers": [sched.state_dict()], "epoch": epoch, "global_step": global_step, "hyper_parameters": cfg}, path)


def load_checkpoint(path, nets, opt=None, sched=None):
    """partial_enc.* and model.* parameters into `nets`, and with `opt` / `sched` their states too; returns the checkpoint dict"""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    sd = {k: v for k, v in ckpt["state_dict"].items() if k.startswith(("partial_enc.", "model."))}
    if not sd:
        raise ValueError(f"{path}: no partial_enc.* / model.* parameters")
    nets.load_state_dict(sd)
    if opt is not None:
        opt.load_state_dict(ckpt["optimizer_states"][0])
        sched.load_state_dict(ckpt["lr_schedulers"][0])
    return ckpt


@click.command()
@click.option("--config", "-c", type=str, default="config/config.yaml", help="path to the reference's config file (.yaml)")
@click.option("--weights", "-w", type=str, default=None, help="start from these weights (.ckpt) without resuming training")
@click.option("--checkpoint", "-ckpt", type=str, default=None, help="resume training from this checkpoint (.ckpt)")
@click.option("--out", type=str, default=None, help="checkpoint directory (default experiments/<experiment.id>/checkpoints)")
@click.option("--max-steps", type=int, default=None, help="stop this run after this many optimiser steps")
@click.option("--device-rng", is_flag=True, help="draw the samples' numpy randn / torch randperm on the GPU, bit for bit (lidiff_b200.rng; also data.device_rng: true in the config)")
def main(config, weights, checkpoint, out, max_steps, device_rng):
    set_deterministic()
    run = ddp.start()
    with open(config) as f:
        cfg = yaml.safe_load(f)
    if os.environ.get("TRAIN_DATABASE"):
        cfg["data"]["data_dir"] = os.environ["TRAIN_DATABASE"]
    cfg["data"].setdefault("dataset_norm", False)
    cfg["data"].setdefault("std_axis_norm", False)
    if run.distributed:
        cfg["train"]["n_gpus"] = run.world
    device = run.device
    out = out or os.path.join("experiments", cfg["experiment"]["id"], "checkpoints")
    os.makedirs(out, exist_ok=True)
    somac = sqrt_one_minus_alphas_cumprod(cfg)
    nets = DiffusionNets(cfg).to(device)
    opt, sched = make_optimizer(nets, cfg)
    first_epoch, step = 0, 0
    if checkpoint is not None:
        ckpt = load_checkpoint(checkpoint, nets, opt, sched)
        first_epoch, step = int(ckpt["epoch"]) + 1, int(ckpt["global_step"])
    elif weights is not None:
        load_checkpoint(weights, nets)
    model, nets = ddp.wrap(nets, run)
    model.train()
    if run.main:
        print("TRAINING MODE")
    dm = TemporalKittiDataModule(cfg, device=device, device_rng=True if device_rng else None)
    train_loader = ddp.sharded(dm.train_dataloader(), run, shuffle=True)
    val_loader = ddp.sharded(dm.val_dataloader(), run, shuffle=False)
    last_step = None if max_steps is None else step + max_steps
    for epoch in range(first_epoch, int(cfg["train"]["max_epoch"])):
        ddp.set_epoch(train_loader, epoch)
        ddp.set_epoch(val_loader, epoch)
        for batch in train_loader:
            log = train_step(model, opt, batch, cfg, somac, device)
            means = ddp.mean_over_ranks([log[k] for k in LOGGED], run, device)
            if run.main:
                print(f"epoch {epoch} step {step}" + ("" if not log["uncond"] else " (unconditional)") + " "
                      + " ".join(f"train/{k}: {v:.9g}" for k, v in zip(LOGGED, means)))
            step += 1
            if step == last_step:
                break
        end_epoch(sched, epoch)
        if (epoch + 1) % VAL_EVERY == 0 and step != last_step:
            val = ddp.mean_over_ranks(validate(nets, next(iter(val_loader)), cfg, device), run, device)
            if run.main:
                print(f"epoch {epoch} " + " ".join(f"val/{k}: {v:.9g}" for k, v in zip(("cd_mean", "cd_std", "precision", "recall", "fscore"), val)))
        path = checkpoint_path(out, cfg, epoch)
        if run.distributed:
            torch.distributed.barrier()
        if run.main:
            save_checkpoint(path, nets, opt, sched, cfg, epoch, step)
            print(f"saved {path}")
        if step == last_step:
            break
    ddp.finish(run)


if __name__ == "__main__":
    main()
