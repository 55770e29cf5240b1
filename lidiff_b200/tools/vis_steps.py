"""Denoising-trajectory strips — the picture of the reference's README figure (`media/diff_steps.png`: the scan, P^T, P^t, P^0)
for one scan, rendered on the GPU (lidiff_b200.render) from the fused engine's trajectory:

    python -m lidiff_b200.tools.vis_steps -d diff.ckpt -r refine.ckpt --scan 000123.ply -T 50 -s 6 --steps 0,10,25,50 --out strip.png
    python -m lidiff_b200.tools.vis_steps --random-weights --scan scan.bin --steps 0,25,50        # no checkpoints at hand

Panels, left to right, with one camera and one z range fitted on the preprocessed (conditioning) scan: that scan; x_t after k
denoising steps for every k of --steps (k = 0: the noisy start, k = T: the loop's output); the post-processed diffusion cloud;
the refined cloud.  The snapshots are device copies of x_t taken between steps (DenoiseEngine.run(snapshot_steps=...)), so the
trajectory is the one complete_scan(..., fresh=True) runs, step graphs included."""
from __future__ import annotations

import click
import numpy as np
import torch

from ..render import Camera, finite_bounds, render, write_png
from .diff_completion_pipeline import load_pcd


def parse_steps(text: str | None, T: int) -> list[int]:
    """the step counts of --steps ("0,10,25,50"; default 0, T/5, T/2, T), ascending without duplicates, each in [0, T]"""
    if text is None or text.strip() == "":
        return sorted({0, T // 5, T // 2, T})
    try:
        steps = [int(t) for t in text.split(",") if t.strip() != ""]
    except ValueError:
        raise ValueError(f"--steps: expected comma-separated integers, got {text!r}")
    if not steps:
        raise ValueError("--steps: no step given")
    bad = [k for k in steps if not 0 <= k <= T]
    if bad:
        raise ValueError(f"--steps: {bad} outside [0, {T}] (T = the number of denoising steps)")
    return sorted(set(steps))


def trajectory(pipe, scan, steps, start_noise=None, step_noise=None) -> dict:
    """the panels' clouds of one raw scan (n, 3): {"scan": preprocessed scan, "steps": {k: x_t after k steps}, "post", "refined"},
    device tensors; the same trajectory as pipe.complete_scan(scan, start_noise, step_noise, fresh=True)"""
    pre = pipe.preprocess_scan(scan).to(pipe.device)
    if start_noise is None:
        start_noise = torch.randn(pre.shape, device=pipe.device)
    x_feats = pre + start_noise.to(pipe.device)
    pipe._last_batch = 1
    refined, post, snaps = pipe.engine().complete(pre, x_feats, step_noise, fresh=True, snapshot_steps=steps)
    return {"scan": pre.reshape(-1, 3), "steps": snaps, "post": post, "refined": refined}


def strip(panels: list, camera: Camera, z_range, point_size: float = 2.0) -> torch.Tensor:
    """the clouds rendered side by side with one camera and z range -> (height, len(panels) width, 3) uint8 device tensor"""
    return torch.cat([render(p, camera, point_size=point_size, z_range=z_range) for p in panels], dim=1)


def panels_of(traj: dict) -> list:
    return [traj["scan"]] + [traj["steps"][k] for k in sorted(traj["steps"])] + [traj["post"], traj["refined"]]


@click.command()
@click.option("--diff", "-d", type=str, default=None, help="path to the diffusion checkpoint")
@click.option("--refine", "-r", type=str, default=None, help="path to the refinement checkpoint")
@click.option("--scan", type=str, required=True, help="the scan (.ply / .bin)")
@click.option("--denoising_steps", "-T", type=click.IntRange(min=1), default=50, help="number of denoising steps")
@click.option("--cond_weight", "-s", type=float, default=6.0, help="conditioning weight")
@click.option("--steps", type=str, default=None, help="step counts to show, e.g. 0,10,25,50 (default: 0, T/5, T/2, T)")
@click.option("--out", "-o", type=str, default="strip.png", help="PNG to write")
@click.option("--width", type=click.IntRange(min=1), default=480, help="width of one panel in pixels")
@click.option("--height", type=click.IntRange(min=1), default=360, help="height of one panel in pixels")
@click.option("--point-size", type=float, default=2.0, help="side of a point's square in pixels")
@click.option("--seed", type=int, default=0, help="seed of torch's generator (the start and step noise)")
@click.option("--random-weights", is_flag=True, help="seeded random parameters instead of checkpoints (plumbing)")
def main(diff, refine, scan, denoising_steps, cond_weight, steps, out, width, height, point_size, seed, random_weights):
    if not random_weights and (diff is None or refine is None):
        raise click.UsageError("give both checkpoints (-d and -r) or --random-weights")
    try:
        ks = parse_steps(steps, denoising_steps)
    except ValueError as e:
        raise click.UsageError(str(e))
    raw = np.asarray(load_pcd(scan), dtype=np.float64)
    from ..pipeline import DiffCompletion
    device = torch.device("cuda", torch.cuda.current_device())
    if random_weights:
        from ..weights import random_state_dict
        sds = {k: random_state_dict(k, i) for i, k in enumerate(("enc", "diff", "refine"))}
        pipe = DiffCompletion(state_dicts=sds, denoising_steps=denoising_steps, cond_weight=cond_weight, device=device)
    else:
        pipe = DiffCompletion(diff, refine, denoising_steps, cond_weight, device=device)
    torch.manual_seed(seed)
    traj = trajectory(pipe, raw, ks)
    lo, hi = finite_bounds(traj["scan"])
    cam = Camera.fit(traj["scan"], width=width, height=height)
    rgb = strip(panels_of(traj), cam, (float(lo[2]), float(hi[2])), point_size)
    write_png(out, rgb)
    click.echo(f"{scan}: panels scan, " + ", ".join(f"x_t after {k} steps" for k in ks) + f", post, refined -> {out}")


if __name__ == "__main__":
    main()
