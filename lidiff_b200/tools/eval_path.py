"""Scores completed scans of a sequence — counterpart of the reference's
`python lidiff/utils/eval_path.py -p PATH [-d diff.ckpt -r refine.ckpt -t 50 -s 6.0]` (lidiff/utils/eval_path.py:65-170): same
options, the same per-scan lines and the same `res_log.yaml` (a JSON dict with jsd, jsd_noclip_3d, rmse_mean, rmse_std, ious,
cd_mean, cd_std, pr, re, f1) next to --path, with every metric computed on the GPU (lidiff_b200.metrics).

    python -m lidiff_b200.tools.eval_path -p results/exp/refine/ --data ./Datasets/SemanticKITTI/dataset/sequences/08
    torchrun --nproc-per-node 8 -m lidiff_b200.tools.eval_path -p results/exp/ -d diff.ckpt -r refine.ckpt

Two modes: with -d / -r (or --random-weights) every scan is completed with lidiff_b200.pipeline.DiffCompletion and the refined
cloud is scored (--cloud diff scores the diffusion-only cloud); without them the `<stem>.ply` files in --path are scored, as
lidiff_b200.tools.diff_completion_pipeline writes them.  With --mesh those files are triangle meshes (io.read_triangle_mesh), each
turned into 1 000 000 points by Metrics3D.convert_to_pcd (open3d's sample_points_uniformly, on the GPU) from the std::mt19937 seeded
with --seed plus the scan's index in the sorted listing, so the samples do not depend on the number of ranks.  Under torchrun scan b runs on rank b mod R; rank 0 folds the per-scan
records in scan order, so the results do not depend on the number of ranks.  --batch-size B completes a rank's scans B at a
time (DiffCompletion.complete_scans); res_log.yaml has the same layout as with B = 1.
"""
from __future__ import annotations

import json
import os

import click
import numpy as np
import torch

from .. import metrics as M
from ..kitti import load_poses, natural_sorted, parse_calibration  # noqa: F401  (part of this module's interface)
from ..sharding import batches_of_rank, gather_scans
from ..shims.open3d.geometry import PointCloud, VoxelGrid
from ..synth import read_ply_xyz

PATH_DATA = "./Datasets/SemanticKITTI/dataset/sequences/08"


def ground_truth(pose: np.ndarray, cur_scan: np.ndarray, seq_map: np.ndarray, max_range: float) -> np.ndarray:
    """the map points within max_range of the pose, in the scan's frame, z in (-4, 4.4), inside the 10 m voxels the scan occupies"""
    d = np.sum((seq_map - pose[:-1, -1]) ** 2, axis=-1) ** 0.5
    gt = seq_map[d < max_range]
    gt = (np.concatenate([gt, np.ones((gt.shape[0], 1))], -1) @ np.linalg.inv(pose).T)[:, :3]
    gt = gt[(gt[:, 2] > -4.0) & (gt[:, 2] < 4.4)]
    view = VoxelGrid.create_from_point_cloud(PointCloud(cur_scan), voxel_size=10.0)
    return gt[np.asarray(view.check_if_included(gt), dtype=bool)]


def scan_completion(data: str, scan_name: str, path: str, pipe, max_range: float, cloud: str):
    """(prediction, the scan's points within max_range)"""
    return scan_completions(data, [scan_name], path, pipe, max_range, cloud)[0]


def read_mesh_prediction(path: str, seed: int) -> np.ndarray:
    """the points Metrics3D.convert_to_pcd samples from the triangle mesh at `path`, with the global stream seeded with `seed`"""
    from ..mesh import STREAM
    from ..shims.open3d.io import read_triangle_mesh
    STREAM.seed(seed)
    return np.asarray(M.Metrics3D.convert_to_pcd(read_triangle_mesh(path)).points)


def scan_completions(data: str, scan_names: list, path: str, pipe, max_range: float, cloud: str, batched: bool = False,
                     mesh_seeds: list | None = None):
    """[(prediction, the scan's points within max_range)] of a group of scans; batched: completed by complete_scans (one
    trajectory per scan, a group shorter than the others starts fresh), else one by one by complete_scan; mesh_seeds (files
    only): the predictions are triangle meshes, sampled with these seeds"""
    points = [np.fromfile(os.path.join(data, "velodyne", s), dtype=np.float32).reshape(-1, 4) for s in scan_names]
    curs = [p[np.sqrt(np.sum(p[:, :3] ** 2, axis=-1)) < max_range, :3] for p in points]
    if pipe is None and mesh_seeds is not None:
        preds = [read_mesh_prediction(os.path.join(path, f"{s.split('.')[0]}.ply"), seed) for s, seed in zip(scan_names, mesh_seeds)]
        preds = [p[np.sqrt(np.sum(p ** 2, axis=-1)) < max_range] for p in preds]
    elif pipe is None:
        preds = [read_ply_xyz(os.path.join(path, f"{s.split('.')[0]}.ply")) for s in scan_names]
        preds = [p[np.sqrt(np.sum(p ** 2, axis=-1)) < max_range] for p in preds]
    else:
        done = pipe.complete_scans(points) if batched else [pipe.complete_scan(p) for p in points]
        preds = [refined if cloud == "refine" else diff for refined, diff in done]
    return list(zip(preds, curs))


def score_scans(data: str, path: str, pipe, max_range: float, cloud: str, device, rank: int = 0, world: int = 1, batch: int = 1,
                mesh_seed: int | None = None):
    """(number of scans, {scan index: record as rows}) for the scans of this rank, completed `batch` at a time; mesh_seed: the
    predictions are triangle meshes, scan b sampled with seed mesh_seed + b"""
    poses = load_poses(os.path.join(data, "calib.txt"), os.path.join(data, "poses.txt"))
    seq_map = np.load(os.path.join(data, "map_clean.npy"))
    scans = natural_sorted(os.listdir(os.path.join(data, "velodyne")))
    n = min(len(poses), len(scans))
    local = {}
    for group in batches_of_rank(n, world, rank, batch):
        seeds = None if mesh_seed is None else [mesh_seed + b for b in group]
        for b, (pred, cur) in zip(group, scan_completions(data, [scans[b] for b in group], path, pipe, max_range, cloud, batch > 1, seeds)):
            gt = ground_truth(poses[b], cur, seq_map, max_range)
            local[b] = M.record_to_rows(M.evaluate_scan(gt, pred, device=device))
    return n, local


def fold(records: dict, verbose: bool = True) -> dict:
    """the metrics over the scans' records in scan order -> the res_log dict (prints the per-scan lines when verbose)"""
    rmse, cd = M.RMSE(), M.ChamferDistance()
    pr = M.PrecisionRecall(*M.PR_ARGS)
    iou = M.CompletionIoU()
    jsd_3d, jsd_bev = [], []
    for b in sorted(records):
        rec = records[b]
        jsd_3d.append(rec.jsd_3d)
        jsd_bev.append(rec.jsd_bev)
        for acc in (rmse, iou, cd, pr):
            acc.add(rec)
        if verbose:
            print(f"JSD 3D: {jsd_3d[-1]}")
            print(f"JSD BEV: {jsd_bev[-1]}")
            _print_totals(rmse, iou, cd, pr)
    res = _totals(rmse, iou, cd, pr)
    return {"jsd": np.array(jsd_bev).mean(), "jsd_noclip_3d": np.array(jsd_3d).mean(), "rmse_mean": res["rmse"][0], "rmse_std": res["rmse"][1],
            "ious": res["ious"], "cd_mean": res["cd"][0], "cd_std": res["cd"][1], "pr": res["auc"][0], "re": res["auc"][1], "f1": res["auc"][2]}


def _totals(rmse, iou, cd, pr):
    return {"rmse": rmse.compute(), "ious": iou.compute(), "cd": cd.compute(), "auc": pr.compute_auc()}


def _print_totals(rmse, iou, cd, pr):
    t = _totals(rmse, iou, cd, pr)
    print(f"RMSE Mean: {t['rmse'][0]}\tRMSE Std: {t['rmse'][1]}")
    for v_size, v in t["ious"].items():
        print(f"Voxel {v_size}cm IOU: {v}")
    print(f"CD Mean: {t['cd'][0]}\tCD Std: {t['cd'][1]}")
    print(f"Precision: {t['auc'][0]}\tRecall: {t['auc'][1]}\tF-Score: {t['auc'][2]}")


def to_json(obj):
    if isinstance(obj, dict):
        return {str(k): to_json(v) for k, v in obj.items()}
    return float(obj)


def log_path(path: str) -> str:
    """res_log.yaml in the directory of --path (its last component dropped, as the reference does)"""
    return os.path.join(os.path.dirname(path) or ".", "res_log.yaml")


@click.command()
@click.option("--path", "-p", type=str, default="", help="path to the scan sequence (the .ply predictions when scoring files)")
@click.option("--voxel_size", "-v", type=float, default=0.05, help="voxel size")
@click.option("--max_range", "-m", type=float, default=50, help="max range")
@click.option("--denoising_steps", "-t", type=int, default=50, help="number of denoising steps")
@click.option("--cond_weight", "-s", type=float, default=6.0, help="conditioning weights")
@click.option("--diff", "-d", type=str, default=None, help="run diffusion pipeline")
@click.option("--refine", "-r", type=str, default=None, help="path to the checkpoint for refinement net")
@click.option("--random-weights", is_flag=True, help="complete with seeded random parameters instead of checkpoints (plumbing)")
@click.option("--data", type=str, default=PATH_DATA, help="sequence directory: velodyne/*.bin, calib.txt, poses.txt, map_clean.npy")
@click.option("--cloud", type=click.Choice(["refine", "diff"]), default="refine", help="which completed cloud to score")
@click.option("--batch-size", type=click.IntRange(min=1), default=1, help="scans completed together per denoising loop (default: 1)")
@click.option("--mesh", is_flag=True, help="the .ply predictions are triangle meshes: score 1 000 000 points sampled from each surface")
@click.option("--seed", type=click.IntRange(min=0), default=0, help="with --mesh: scan b is sampled with std::mt19937(seed + b)")
def main(path, voxel_size, max_range, denoising_steps, cond_weight, diff, refine, random_weights, data, cloud, batch_size, mesh, seed):
    if mesh and (random_weights or diff is not None or refine is not None):
        raise click.UsageError("--mesh scores mesh files; it cannot be combined with -d / -r / --random-weights")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(device)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    pipe = None
    if random_weights:
        from ..pipeline import DiffCompletion
        from ..weights import random_state_dict
        sds = {k: random_state_dict(k, i) for i, k in enumerate(("enc", "diff", "refine"))}
        pipe = DiffCompletion(state_dicts=sds, denoising_steps=denoising_steps, cond_weight=cond_weight, device=device)
    elif diff is not None or refine is not None:
        from ..pipeline import DiffCompletion
        pipe = DiffCompletion(diff, refine, denoising_steps, cond_weight, device=device)
    n, local = score_scans(data, path, pipe, max_range, cloud, device, rank, world, batch_size, seed if mesh else None)
    gathered = gather_scans(local, n, device)
    if rank == 0:
        res = fold({b: M.record_from_rows(rows) for b, rows in gathered.items()})
        print("\n\n=================== FINAL RESULTS ===================\n\n")
        print(f"JSD 3D: {res['jsd_noclip_3d']}")
        print(f"JSD BEV: {res['jsd']}")
        print(f"RMSE Mean: {res['rmse_mean']}\tRMSE Std: {res['rmse_std']}")
        for v_size, v in res["ious"].items():
            print(f"Voxel {v_size}cm IOU: {v}")
        print(f"CD Mean: {res['cd_mean']}\tCD Std: {res['cd_std']}")
        print(f"Precision: {res['pr']}\tRecall: {res['re']}\tF-Score: {res['f1']}")
        with open(log_path(path), "w") as f:
            json.dump(to_json(res), f)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
