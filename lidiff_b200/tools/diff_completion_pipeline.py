"""Command-line scene completion — counterpart of the reference's
`python3 tools/diff_completion_pipeline.py -d diff_net.ckpt -r refine_net.ckpt -T 50 -s 6.0`
(/root/reference/lidiff/tools/diff_completion_pipeline.py:179-212): same options, same outputs
(`results/<exp>/{diff,refine}/<scan>.ply`; with `--normals` each PLY also carries the reference's open3d estimate_normals()
normals as `nx ny nz`, computed on the GPU by lidiff_b200.normals), plus sharding of the scans over the ranks of a torchrun job
(one process per GPU, scan b on rank b mod R; SURVEY.md 8e).  --batch-size B completes a rank's scans B at a time
(DiffCompletion.complete_scans: one trajectory per scan, every launch shared); the files written are the same as with B = 1.
With --ssc each refined cloud is also written as a SemanticKITTI scene-completion grid, `results/<exp>/ssc/<scan>.bin` (the 0.2 m
256 x 256 x 32 occupancy of lidiff_b200.ssc, voxelized on the GPU), which `eval_path --voxels` and SSC tools read.

    torchrun --nproc-per-node 8 -m lidiff_b200.tools.diff_completion_pipeline -d diff.ckpt -r refine.ckpt --path ./Datasets/test
    python -m lidiff_b200.tools.diff_completion_pipeline --random-weights --path ./Datasets/test     # no checkpoints at hand
"""
from __future__ import annotations

import os
import time

import click
import numpy as np
import torch

from ..normals import estimate_normals
from .. import ssc as S
from ..pipeline import DiffCompletion
from ..sharding import batches_of_rank
from ..synth import read_ply_xyz


def load_pcd(pcd_file: str) -> np.ndarray:
    if pcd_file.endswith(".bin"):
        return np.fromfile(pcd_file, dtype=np.float32).reshape((-1, 4))[:, :3]
    if pcd_file.endswith(".ply"):
        return read_ply_xyz(pcd_file)
    raise click.ClickException(f"Point cloud format '.{pcd_file.split('.')[-1]}' not supported. (supported formats: .bin (kitti format), .ply)")


def write_ply(path: str, pts: np.ndarray, normals: np.ndarray | None = None):
    """binary little-endian PLY of fp64 `x y z` vertices, or `x y z nx ny nz` with `normals` (the layout open3d writes)"""
    pts = np.ascontiguousarray(pts, dtype=np.float64)
    props = "property double x\nproperty double y\nproperty double z\n"
    if normals is not None:
        normals = np.asarray(normals, dtype=np.float64)
        if normals.shape != pts.shape:
            raise ValueError(f"write_ply: normals of shape {normals.shape} for points of shape {pts.shape}")
        pts = np.concatenate([pts, normals], 1)
        props += "property double nx\nproperty double ny\nproperty double nz\n"
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\ncomment Created by lidiff_b200\n"
                 f"element vertex {pts.shape[0]}\n{props}end_header\n").encode("ascii"))
        f.write(pts.astype("<f8").tobytes())


@click.command()
@click.option("--diff", "-d", type=str, default="checkpoints/diff_net.ckpt", help="path to the diffusion checkpoint")
@click.option("--refine", "-r", type=str, default="checkpoints/refine_net.ckpt", help="path to the refinement checkpoint")
@click.option("--denoising_steps", "-T", type=int, default=50, help="number of denoising steps (default: 50)")
@click.option("--cond_weight", "-s", type=float, default=6.0, help="conditioning weight (default: 6.0)")
@click.option("--path", type=str, default="./Datasets/test/", help="directory with .ply / .bin scans")
@click.option("--out", type=str, default="./results", help="output root")
@click.option("--random-weights", is_flag=True, help="seeded random parameters instead of checkpoints (plumbing / benchmarking)")
@click.option("--normals", is_flag=True, help="write open3d's estimate_normals() (30 nearest neighbours) as nx ny nz, as the reference does")
@click.option("--batch-size", type=click.IntRange(min=1), default=1, help="scans completed together per denoising loop (default: 1)")
@click.option("--ssc", is_flag=True, help="also write each refined cloud as a SemanticKITTI scene-completion grid, ssc/<scan>.bin")
def main(diff, refine, denoising_steps, cond_weight, path, out, random_weights, normals, batch_size, ssc):
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    exp_dir = diff.split("/")[-1].split(".")[0].replace("=", "") + f"_T{denoising_steps}_s{cond_weight}"
    if random_weights:
        from ..weights import random_state_dict
        sds = {k: random_state_dict(k, i) for i, k in enumerate(("enc", "diff", "refine"))}
        pipe = DiffCompletion(state_dicts=sds, denoising_steps=denoising_steps, cond_weight=cond_weight, device=device)
    else:
        pipe = DiffCompletion(diff, refine, denoising_steps, cond_weight, device=device)
    os.makedirs(f"{out}/{exp_dir}/refine", exist_ok=True)
    os.makedirs(f"{out}/{exp_dir}/diff", exist_ok=True)
    if ssc:
        os.makedirs(f"{out}/{exp_dir}/ssc", exist_ok=True)
    files = sorted(os.listdir(path), key=lambda s: [int(t) if t.isdigit() else t for t in __import__("re").split(r"(\d+)", s)])
    for group in batches_of_rank(len(files), world, rank, batch_size):
        names = [files[i] for i in group]
        points = [load_pcd(os.path.join(path, name)) for name in names]
        start = time.time()
        results = [pipe.complete_scan(points[0])] if batch_size == 1 else pipe.complete_scans(points)
        torch.cuda.synchronize()
        print(f"[rank {rank}] {', '.join(names)}: took {time.time() - start:.3f}s")
        for name, (refine_scan, diff_scan) in zip(names, results):
            stem = name.split(".")[0]
            for kind, cloud in (("refine", refine_scan), ("diff", diff_scan)):
                nrm = estimate_normals(cloud, device=device).cpu().numpy() if normals else None
                write_ply(f"{out}/{exp_dir}/{kind}/{stem}.ply", cloud, nrm)
            if ssc:
                S.write_bin(f"{out}/{exp_dir}/ssc/{stem}.bin", S.voxelize(refine_scan, device=device)[0])
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
