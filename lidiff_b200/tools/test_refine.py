"""The refinement network's test mode on SemanticKITTI — counterpart of the reference's `python train_refine.py -w refine.ckpt --test
-c config_refine.yaml` (lidiff/train_refine.py -> RefineDiffusion.test_step / validation_step, lidiff/models/models_refine.py:78-134),
single process, without the open3d viewer.

For every batch of the loader (`test`: the TRAIN sequences with split 'validation', as the reference's test_dataloader; `val`:
sequence 08), the noisy rows are voxelised at the config's resolution over all four batched columns, the refinement MinkUNet predicts
up_factor offsets per row, and the Chamfer distance of the refined rows to `pcd_full` (pytorch3d's, lidiff_b200.metrics) is printed
per batch and as the mean at the end.  With --out the refined cloud and its normals are written to
<out>/refined/<seq>/<first stem of the window>.ply.

    python -m lidiff_b200.tools.test_refine -w refine.ckpt -c lidiff/config/config_refine.yaml --out experiments/refine
    python -m lidiff_b200.tools.test_refine --random-weights -c config_refine.yaml --loader val      # no checkpoint at hand
"""
from __future__ import annotations

import os

import click
import numpy as np
import torch
import yaml

from .. import me as ME
from ..datasets_refine import TemporalKittiDataModule
from ..metrics import chamfer_distance
from ..minkunet import MinkUNet
from ..normals import estimate_normals
from .diff_completion_pipeline import write_ply
from .test_completion import set_deterministic

MAX_BATCH = 51          # round(b / resolution) = 20 b must stay within the coordinate keys' 10 batch bits


def load_refine_net(weights, up_factor: int, device, random_weights: bool = False) -> MinkUNet:
    """MinkUNet(3, 3 up_factor) from the checkpoint's model_refine.* parameters (or seeded random ones), in eval mode"""
    net = MinkUNet(in_channels=3, out_channels=3 * up_factor)
    if random_weights:
        from ..weights import random_state_dict
        sd = random_state_dict("refine", 2) if up_factor == 6 else net.state_dict()
    else:
        ckpt = torch.load(weights, map_location="cpu", weights_only=False)
        sd = {k[len("model_refine."):]: v for k, v in ckpt["state_dict"].items() if k.startswith("model_refine.")}
        if not sd:
            raise ValueError(f"{weights}: no model_refine.* parameters")
    net.load_state_dict(sd)
    return net.to(device).eval()


@torch.no_grad()
def refine_batch(net, batch, resolution: float, up_factor: int, device):
    """validation_step's arithmetic (models_refine.py:103-123): (refined (B, up_factor N, 3) float32, Chamfer loss)"""
    b = batch["pcd_noise"].shape[0]
    if b > MAX_BATCH:
        raise ValueError(f"batch of {b} clouds: the refinement path keys the batch column as round(b / {resolution:g}); at most "
                         f"{MAX_BATCH} clouds fit")
    x_feats = ME.utils.batched_coordinates(list(batch["pcd_noise"]), dtype=torch.float32, device=device)
    x_coord = torch.round(x_feats / resolution)
    x_feats = x_feats[:, 1:]
    x_t = ME.TensorField(features=x_feats, coordinates=x_coord, quantization_mode=ME.SparseTensorQuantizationMode.UNWEIGHTED_AVERAGE,
                         minkowski_algorithm=ME.MinkowskiAlgorithm.SPEED_OPTIMIZED, device=device)
    offset = net(x_t).reshape(-1, up_factor, 3)
    refined = (x_feats[:, None, :] + offset).reshape(batch["pcd_full"].shape[0], -1, 3)
    loss, _ = chamfer_distance(refined, batch["pcd_full"].to(device))
    return refined, loss


def ply_path(out: str, window) -> str:
    first = window[0]
    seq_dir = os.path.join(out, "refined", first.split("/")[-3])
    os.makedirs(seq_dir, exist_ok=True)
    return os.path.join(seq_dir, os.path.basename(first).split(".")[0] + ".ply")


@click.command()
@click.option("--weights", "-w", type=str, default=None, help="path to the refinement checkpoint (.ckpt)")
@click.option("--config", "-c", type=str, default="config/config_refine.yaml", help="path to the reference's refine config (.yaml)")
@click.option("--loader", type=click.Choice(["test", "val"]), default="test", help="test_dataloader (as --test runs) or val_dataloader")
@click.option("--out", type=str, default=None, help="write <out>/refined/<seq>/<stem>.ply with normals")
@click.option("--random-weights", is_flag=True, help="seeded random parameters instead of a checkpoint (plumbing / benchmarking)")
def main(weights, config, loader, out, random_weights):
    set_deterministic()
    with open(config) as f:
        cfg = yaml.safe_load(f)
    if os.environ.get("TRAIN_DATABASE"):
        cfg["data"]["data_dir"] = os.environ["TRAIN_DATABASE"]
    if weights is None and not random_weights:
        raise click.UsageError("give a checkpoint with -w or pass --random-weights")
    device = torch.device("cuda", torch.cuda.current_device())
    up = int(cfg["train"]["up_factor"])
    res = float(cfg["data"]["resolution"])
    net = load_refine_net(weights, up, device, random_weights)
    dm = TemporalKittiDataModule(cfg, device=device)
    data = dm.test_dataloader() if loader == "test" else dm.val_dataloader()
    tag = "test" if loader == "test" else "val"
    losses = []
    for i, batch in enumerate(data):
        refined, loss = refine_batch(net, batch, res, up, device)
        losses.append(loss.item())
        print(f"batch {i} {tag}/cd_loss: {losses[-1]:.9g}")
        if out is not None:
            for b, window in enumerate(batch["filename"]):
                pts = refined[b].double()
                write_ply(ply_path(out, window), pts.cpu().numpy(), estimate_normals(pts, device=device).cpu().numpy())
    print(f"{tag}/cd_loss mean over {len(losses)} batches: {float(np.mean(losses)) if losses else float('nan'):.9g}")


if __name__ == "__main__":
    main()
