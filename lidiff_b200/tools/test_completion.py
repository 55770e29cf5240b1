"""The diffusion network's test mode on SemanticKITTI — counterpart of the reference's `python train.py -w diff.ckpt --test -c
config.yaml` (lidiff/train.py:16-20,116-118 -> DiffusionPoints.test_step, lidiff/models/models.py:264-335), single process.

For every batch of the validation sequences (`test_dataloader`: split 'validation', the config's batch size) the partial scans are
completed from themselves (`pcd_part` tiled 10 times, models.py:290) with DiffCompletion.complete_scans(preprocessed=True), whose
multistep state carries across batches as the reference's scheduler does; the diffusion output after the reference's
post-processing is written to `<out>/generated_pcd/<seq>/<stem>.ply`, and Chamfer distance and precision / recall against `pcd_full`
are accumulated and printed after every batch.  A batch whose PLYs all exist is skipped (valid_paths).

    python -m lidiff_b200.tools.test_completion -w diff.ckpt -c lidiff/config/config.yaml --out experiments/run
    python -m lidiff_b200.tools.test_completion --random-weights -c config.yaml -T 5       # no checkpoint at hand
"""
from __future__ import annotations

import os

import click
import numpy as np
import torch
import yaml

from ..datasets import TemporalKittiDataModule
from ..metrics import ChamferDistance, PrecisionRecall
from ..pipeline import DiffCompletion
from .diff_completion_pipeline import write_ply


def set_deterministic():
    """lidiff/train.py:16-20"""
    np.random.seed(42)
    torch.manual_seed(42)
    torch.cuda.manual_seed(42)
    torch.backends.cudnn.deterministic = True


def valid_paths(out: str, filenames):
    """(every output already written, output paths) of a batch (models.py:264-276)"""
    paths, skip = [], []
    for fname in filenames:
        seq_dir = os.path.join(out, "generated_pcd", fname.split("/")[-3])
        os.makedirs(seq_dir, exist_ok=True)
        paths.append(os.path.join(seq_dir, fname.split("/")[-1].split(".")[0] + ".ply"))
        skip.append(os.path.isfile(paths[-1]))
    return bool(np.all(skip)), paths


@click.command()
@click.option("--weights", "-w", type=str, default=None, help="path to the diffusion checkpoint (.ckpt)")
@click.option("--config", "-c", type=str, default="config/config.yaml", help="path to the reference's config file (.yaml)")
@click.option("--out", type=str, default="./experiments", help="output root: <out>/generated_pcd/<seq>/<scan>.ply")
@click.option("--random-weights", is_flag=True, help="seeded random parameters instead of a checkpoint (plumbing / benchmarking)")
@click.option("--denoising_steps", "-T", type=int, default=None, help="number of denoising steps (default: the config's diff.s_steps)")
def main(weights, config, out, random_weights, denoising_steps):
    set_deterministic()
    with open(config) as f:
        cfg = yaml.safe_load(f)
    if os.environ.get("TRAIN_DATABASE"):
        cfg["data"]["data_dir"] = os.environ["TRAIN_DATABASE"]
    cfg["data"].setdefault("dataset_norm", False)
    cfg["data"].setdefault("std_axis_norm", False)
    if weights is None and not random_weights:
        raise click.UsageError("give a checkpoint with -w or pass --random-weights")
    steps = int(denoising_steps or cfg["diff"]["s_steps"])
    device = torch.device("cuda", torch.cuda.current_device())
    hp = {"data": {"resolution": cfg["data"]["resolution"], "num_points": cfg["data"]["num_points"]}}
    if random_weights:
        from ..weights import random_state_dict
        sds = {k: random_state_dict(k, i) for i, k in enumerate(("enc", "diff", "refine"))}
        pipe = DiffCompletion(state_dicts=sds, denoising_steps=steps, cond_weight=cfg["train"]["uncond_w"], hparams=hp, device=device)
    else:
        pipe = DiffCompletion(weights, None, steps, cfg["train"]["uncond_w"], hparams=hp, device=device)
    print("TESTING MODE")
    resolution = cfg["data"]["resolution"]
    chamfer, prec_rec = ChamferDistance(), PrecisionRecall(resolution, 2 * resolution, 100)
    for batch in TemporalKittiDataModule(cfg, device=device).test_dataloader():
        skip, paths = valid_paths(out, batch["filename"])
        if skip:
            print(f"Skipping generation from {paths[0]} to {paths[-1]}")
            continue
        results = pipe.complete_scans(batch["pcd_part"].repeat(1, 10, 1), preprocessed=True)
        for i, (_, post) in enumerate(results):
            print(f"Saving {paths[i]}")
            write_ply(paths[i], post)
            gt = batch["pcd_full"][i].double()
            chamfer.update(gt, post)
            prec_rec.update(gt, post)
        cd_mean, cd_std = chamfer.compute()
        pr, re, f1 = prec_rec.compute_auc()
        print(f"CD Mean: {cd_mean}\tCD Std: {cd_std}")
        print(f"Precision: {pr}\tRecall: {re}\tF-Score: {f1}")


if __name__ == "__main__":
    main()
