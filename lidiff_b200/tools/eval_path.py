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
with --seed plus the scan's index in the sorted listing, so the samples do not depend on the number of ranks.  With --voxels
they are SemanticKITTI scene-completion grids (`<stem>.label` or `<stem>.bin`, lidiff_b200.ssc), each scored as its occupied voxels'
centres; only the scans with a grid are scored (the dataset has grids for every 5th scan), in scan order.  --ssc (any prediction
kind) also voxelizes each prediction, before the max_range filter, into the 0.2 m SSC grid and adds the benchmark's completion
IoU / precision / recall against --data's `voxels/<stem>.label` + `.invalid` to the output as ssc_iou, ssc_precision and
ssc_recall; scans without a ground-truth grid do not count.  Under torchrun scan b runs on rank b mod R; rank 0 folds the per-scan
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
from .. import ssc as S
from ..sharding import batches_of_rank, gather_scans, scans_of_rank
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


def grid_file(path: str, scan_name: str) -> str | None:
    """the scene-completion grid predicted for a scan: `<stem>.label`, else `<stem>.bin`, in `path` (None: neither)"""
    for ext in (".label", ".bin"):
        f = os.path.join(path, scan_name.split(".")[0] + ext)
        if os.path.exists(f):
            return f
    return None


def voxel_predictions(files: list, device) -> list:
    """the centres of the occupied voxels of each grid file, converted on the GPU (ssc.grid_points) in one call per kind"""
    grids = [S.read_grid(f) for f in files]
    preds = [None] * len(files)
    for kind in ("labels", "bits"):
        idx = [i for i, (_, k) in enumerate(grids) if k == kind]
        if idx:
            pts, off = S.grid_points([grids[i][0] for i in idx], kind, device=device)
            pts = pts.cpu().numpy()
            for j, i in enumerate(idx):
                preds[i] = pts[off[j]:off[j + 1]]
    return preds


def ssc_counts(data: str, scan_name: str, pred, device) -> np.ndarray:
    """int64 [1, TP, FP, FN] of the prediction voxelized into the SSC grid against `voxels/<stem>.label` + `.invalid` of the
    sequence, or [0, 0, 0, 0] when the scan has no ground-truth grid"""
    stem = os.path.join(data, "voxels", scan_name.split(".")[0])
    if not os.path.exists(stem + ".label"):
        return np.zeros(4, np.int64)
    labels, _ = S.read_grid(stem + ".label")
    bits, _ = S.voxelize(pred, device=device)
    return np.concatenate([[1], S.completion_counts(bits, labels, S.read_invalid(stem + ".invalid"), device=device)]).astype(np.int64)


def ssc_to_rows(counts: np.ndarray) -> torch.Tensor:
    """the 4 int64 of ssc_counts as 3 float32 rows (their raw bytes, padded), appended to a record's rows"""
    words = np.concatenate([np.asarray(counts, np.int64).view(np.float32), np.zeros(1, np.float32)])
    return torch.from_numpy(words.reshape(3, 3).copy())


def ssc_from_rows(rows: torch.Tensor) -> np.ndarray:
    return rows.detach().cpu().contiguous().numpy().astype(np.float32, copy=False).reshape(-1)[:8].view(np.int64).copy()


def _in_range(p: np.ndarray, max_range: float) -> np.ndarray:
    return p[np.sqrt(np.sum(p ** 2, axis=-1)) < max_range]


def _predictions(data: str, scan_names: list, path: str, pipe, max_range: float, cloud: str, batched: bool, mesh_seeds, grid_files,
                 device):
    """(the predictions as read or completed, the scans' points within max_range)"""
    points = [np.fromfile(os.path.join(data, "velodyne", s), dtype=np.float32).reshape(-1, 4) for s in scan_names]
    curs = [p[np.sqrt(np.sum(p[:, :3] ** 2, axis=-1)) < max_range, :3] for p in points]
    if pipe is None and grid_files is not None:
        preds = voxel_predictions(grid_files, device)
    elif pipe is None and mesh_seeds is not None:
        preds = [read_mesh_prediction(os.path.join(path, f"{s.split('.')[0]}.ply"), seed) for s, seed in zip(scan_names, mesh_seeds)]
    elif pipe is None:
        preds = [read_ply_xyz(os.path.join(path, f"{s.split('.')[0]}.ply")) for s in scan_names]
    else:
        done = pipe.complete_scans(points) if batched else [pipe.complete_scan(p) for p in points]
        preds = [refined if cloud == "refine" else diff for refined, diff in done]
    return preds, curs


def scan_completions(data: str, scan_names: list, path: str, pipe, max_range: float, cloud: str, batched: bool = False,
                     mesh_seeds: list | None = None, grid_files: list | None = None, device="cuda"):
    """[(prediction, the scan's points within max_range)] of a group of scans; batched: completed by complete_scans (one
    trajectory per scan, a group shorter than the others starts fresh), else one by one by complete_scan; mesh_seeds (files
    only): the predictions are triangle meshes, sampled with these seeds; grid_files (files only): the predictions are these
    scene-completion grids, scored as their voxel centres.  Predictions read from files keep their points within max_range."""
    preds, curs = _predictions(data, scan_names, path, pipe, max_range, cloud, batched, mesh_seeds, grid_files, device)
    if pipe is None:
        preds = [_in_range(p, max_range) for p in preds]
    return list(zip(preds, curs))


def score_scans(data: str, path: str, pipe, max_range: float, cloud: str, device, rank: int = 0, world: int = 1, batch: int = 1,
                mesh_seed: int | None = None, voxels: bool = False, ssc: bool = False):
    """(number of scored scans, {scored scan index: record as rows}) for the scans of this rank, completed `batch` at a time;
    mesh_seed: the predictions are triangle meshes, scan b sampled with seed mesh_seed + b; voxels: the predictions are
    scene-completion grids, and only the scans with a grid file are scored, numbered 0..m-1 in scan order, sharded and converted
    ssc.CHUNK at a time; ssc: every record's rows end with ssc_to_rows(ssc_counts(...)) of the prediction before the max_range
    filter.  Raises FileNotFoundError when --voxels finds no grid, or --ssc no ground-truth grid, for the scored scans."""
    poses = load_poses(os.path.join(data, "calib.txt"), os.path.join(data, "poses.txt"))
    seq_map = np.load(os.path.join(data, "map_clean.npy"))
    scans = natural_sorted(os.listdir(os.path.join(data, "velodyne")))
    n = min(len(poses), len(scans))
    files = [grid_file(path, scans[b]) for b in range(n)] if voxels else None
    scored = [b for b in range(n) if files[b] is not None] if voxels else list(range(n))
    if voxels and not scored:
        raise FileNotFoundError(f"no <stem>.label or <stem>.bin grid in {path} for the scans of {data}")
    if ssc and not any(os.path.exists(os.path.join(data, "voxels", scans[b].split(".")[0] + ".label")) for b in scored):
        raise FileNotFoundError(f"--ssc: no ground-truth grid voxels/<stem>.label in {data} for the scored scans")
    if voxels:
        mine = scans_of_rank(len(scored), world, rank)
        groups = [mine[i:i + S.CHUNK] for i in range(0, len(mine), S.CHUNK)]
    else:
        groups = batches_of_rank(n, world, rank, batch)
    local = {}
    for group in groups:
        bs = [scored[j] for j in group]
        seeds = None if mesh_seed is None else [mesh_seed + b for b in bs]
        preds, curs = _predictions(data, [scans[b] for b in bs], path, pipe, max_range, cloud, batch > 1, seeds,
                                   [files[b] for b in bs] if voxels else None, device)
        for j, b, pred, cur in zip(group, bs, preds, curs):
            gt = ground_truth(poses[b], cur, seq_map, max_range)
            rows = M.record_to_rows(M.evaluate_scan(gt, _in_range(pred, max_range) if pipe is None else pred, device=device))
            if ssc:
                rows = torch.cat([rows, ssc_to_rows(ssc_counts(data, scans[b], pred, device))])
            local[j] = rows
    return len(scored), local


def fold_ssc(counts: dict) -> dict:
    """the scene-completion scores of the ssc_counts of the scans with ground truth, summed in scan order -> the res_log keys"""
    acc = S.SSCCompletion()
    for b in sorted(counts):
        if counts[b][0]:
            acc.add(counts[b][1:])
    res = acc.compute()
    return {"ssc_iou": res["iou"], "ssc_precision": res["precision"], "ssc_recall": res["recall"]}


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
@click.option("--voxels", is_flag=True, help="the predictions are SemanticKITTI scene-completion grids <stem>.label / <stem>.bin: score "
              "their voxel centres, for the scans that have one")
@click.option("--ssc", is_flag=True, help="also score the predictions' 0.2 m grid occupancy against --data's voxels/<stem>.label + "
              ".invalid: the SSC benchmark's completion IoU / precision / recall")
def main(path, voxel_size, max_range, denoising_steps, cond_weight, diff, refine, random_weights, data, cloud, batch_size, mesh, seed,
         voxels, ssc):
    if mesh and (random_weights or diff is not None or refine is not None):
        raise click.UsageError("--mesh scores mesh files; it cannot be combined with -d / -r / --random-weights")
    if voxels and (mesh or random_weights or diff is not None or refine is not None):
        raise click.UsageError("--voxels scores grid files; it cannot be combined with --mesh / -d / -r / --random-weights")
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
    n, local = score_scans(data, path, pipe, max_range, cloud, device, rank, world, batch_size, seed if mesh else None, voxels, ssc)
    gathered = gather_scans(local, n, device)
    if rank == 0:
        res = fold({b: M.record_from_rows(rows[:-3] if ssc else rows) for b, rows in gathered.items()})
        if ssc:
            res.update(fold_ssc({b: ssc_from_rows(rows[-3:]) for b, rows in gathered.items()}))
        print("\n\n=================== FINAL RESULTS ===================\n\n")
        print(f"JSD 3D: {res['jsd_noclip_3d']}")
        print(f"JSD BEV: {res['jsd']}")
        print(f"RMSE Mean: {res['rmse_mean']}\tRMSE Std: {res['rmse_std']}")
        for v_size, v in res["ious"].items():
            print(f"Voxel {v_size}cm IOU: {v}")
        print(f"CD Mean: {res['cd_mean']}\tCD Std: {res['cd_std']}")
        print(f"Precision: {res['pr']}\tRecall: {res['re']}\tF-Score: {res['f1']}")
        if ssc:
            print(f"SSC IoU: {res['ssc_iou']}\tSSC Precision: {res['ssc_precision']}\tSSC Recall: {res['ssc_recall']}")
        with open(log_path(path), "w") as f:
            json.dump(to_json(res), f)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
