"""Train the refinement network on SemanticKITTI — single-process counterpart of the reference's
`python train_refine.py -c config_refine.yaml [-w W] [-ckpt C]` (lidiff/train_refine.py, RefineDiffusion.training_step /
validation_step / configure_optimizers, lidiff/models/models_refine.py:53-76, 103-139).

Every step runs training_step's arithmetic with gradients: the noisy rows voxelised at the config's resolution, MinkUNet's up_factor
offsets per row, pytorch3d's Chamfer loss against `pcd_full` (lidiff_b200.metrics), backward through the sparse convolutions'
CUDA gradients (lidiff_b200.me) and one Adam step (lr = train.lr, betas (0.9, 0.999), no scheduler).  Every 5 epochs val/cd_loss is
the mean over the first 5 % of the validation batches, as the reference's Trainer (check_val_every_n_epoch=5,
limit_val_batches=0.05).  After every epoch <out>/<experiment.id>_epoch=NN.ckpt holds the Lightning checkpoint fields the
reference and tools/test_refine read: state_dict (model_refine.*), optimizer_states, epoch, global_step, hyper_parameters.

    python -m lidiff_b200.tools.train_refine -c lidiff/config/config_refine.yaml
    python -m lidiff_b200.tools.train_refine -c config_refine.yaml -ckpt experiments/Refine_Up6/checkpoints/Refine_Up6_epoch=02.ckpt
"""
from __future__ import annotations

import os

import click
import torch
import yaml

from ..datasets_refine import TemporalKittiDataModule
from ..minkunet import MinkUNet
from .test_completion import set_deterministic
from .test_refine import refine_batch

# training_step's arithmetic is validation_step's (test_refine.refine_batch) with gradients: the same function without its no_grad
# decorator, so that the two cannot drift apart
refine_forward = refine_batch.__wrapped__

VAL_EVERY = 5
LIMIT_VAL_BATCHES = 0.05


def make_optimizer(net, cfg):
    """configure_optimizers (models_refine.py:136-139)"""
    return torch.optim.Adam(net.parameters(), lr=float(cfg["train"]["lr"]), betas=(0.9, 0.999))


def train_step(net, opt, batch, cfg, device) -> torch.Tensor:
    """one training_step + optimizer step; returns the (detached) Chamfer loss"""
    opt.zero_grad(set_to_none=True)
    _, loss = refine_forward(net, batch, float(cfg["data"]["resolution"]), int(cfg["train"]["up_factor"]), device)
    loss.backward()
    opt.step()
    return loss.detach()


def validate(net, loader, cfg, device) -> float:
    """mean val/cd_loss over the first limit_val_batches of the loader (at least one batch)"""
    n = max(1, int(len(loader) * LIMIT_VAL_BATCHES))
    net.eval()
    losses = []
    for i, batch in enumerate(loader):
        if i == n:
            break
        losses.append(refine_batch(net, batch, float(cfg["data"]["resolution"]), int(cfg["train"]["up_factor"]), device)[1].item())
    net.train()
    return sum(losses) / len(losses)


def checkpoint_path(out: str, cfg, epoch: int) -> str:
    return os.path.join(out, f"{cfg['experiment']['id']}_epoch={epoch:02d}.ckpt")


def save_checkpoint(path, net, opt, cfg, epoch: int, global_step: int):
    torch.save({"state_dict": {f"model_refine.{k}": v.detach().cpu() for k, v in net.state_dict().items()},
                "optimizer_states": [opt.state_dict()], "epoch": epoch, "global_step": global_step, "hyper_parameters": cfg}, path)


def load_checkpoint(path, net, opt=None):
    """model_refine.* parameters into `net`, and with `opt` the optimizer state too; returns the checkpoint dict"""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    sd = {k[len("model_refine."):]: v for k, v in ckpt["state_dict"].items() if k.startswith("model_refine.")}
    if not sd:
        raise ValueError(f"{path}: no model_refine.* parameters")
    net.load_state_dict(sd)
    if opt is not None:
        opt.load_state_dict(ckpt["optimizer_states"][0])
    return ckpt


@click.command()
@click.option("--config", "-c", type=str, default="config/config_refine.yaml", help="path to the reference's refine config (.yaml)")
@click.option("--weights", "-w", type=str, default=None, help="start from these weights (.ckpt) without resuming training")
@click.option("--checkpoint", "-ckpt", type=str, default=None, help="resume training from this checkpoint (.ckpt)")
@click.option("--out", type=str, default=None, help="checkpoint directory (default experiments/<experiment.id>/checkpoints)")
def main(config, weights, checkpoint, out):
    set_deterministic()
    with open(config) as f:
        cfg = yaml.safe_load(f)
    if os.environ.get("TRAIN_DATABASE"):
        cfg["data"]["data_dir"] = os.environ["TRAIN_DATABASE"]
    device = torch.device("cuda", torch.cuda.current_device())
    out = out or os.path.join("experiments", cfg["experiment"]["id"], "checkpoints")
    os.makedirs(out, exist_ok=True)
    net = MinkUNet(in_channels=3, out_channels=3 * int(cfg["train"]["up_factor"])).to(device)
    opt = make_optimizer(net, cfg)
    first_epoch, step = 0, 0
    if checkpoint is not None:
        ckpt = load_checkpoint(checkpoint, net, opt)
        first_epoch, step = int(ckpt["epoch"]) + 1, int(ckpt["global_step"])
    elif weights is not None:
        load_checkpoint(weights, net)
    net.train()
    dm = TemporalKittiDataModule(cfg, device=device)
    train_loader, val_loader = dm.train_dataloader(), dm.val_dataloader()
    for epoch in range(first_epoch, int(cfg["train"]["max_epoch"])):
        for batch in train_loader:
            loss = train_step(net, opt, batch, cfg, device)
            print(f"epoch {epoch} step {step} train/cd_loss: {loss.item():.9g}")
            step += 1
        if (epoch + 1) % VAL_EVERY == 0:
            print(f"epoch {epoch} val/cd_loss: {validate(net, val_loader, cfg, device):.9g}")
        path = checkpoint_path(out, cfg, epoch)
        save_checkpoint(path, net, opt, cfg, epoch, step)
        print(f"saved {path}")


if __name__ == "__main__":
    main()
