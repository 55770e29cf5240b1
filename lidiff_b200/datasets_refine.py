"""The refinement network's SemanticKITTI samples on the GPU — the reference's `TemporalKITTISet`
(lidiff/datasets/dataloader/SemanticKITTITemporalAggr.py), `aggregate_pcds` (lidiff/utils/pcd_preprocess.py),
`point_set_to_sparse_refine` (lidiff/utils/collations.py:20-39) and `TemporalKittiDataModule` (lidiff/datasets/datasets_refine.py).

Per sample, as the reference's __getitem__ (line numbers of SemanticKITTITemporalAggr.py / pcd_preprocess.py):
  * the window's scans (:42-55) are read on the host and uploaded once, the frame scan t_frame = len(window) // 2 last;
    lb2_aggregate_window keeps (label & 0xFFFF) < 252 and the fp32 range > 3.5 m, and applies the scan's pose and then the inverse
    pose of the window's LAST scan (aggregate_pcds leaves `fname` at the last scan of its loop, pcd_preprocess.py:124-126);
  * the training augmentation (:59-67) with its random numbers from numpy's global generator, as lidiff_b200.datasets.augment;
  * the noisy rows (:77-79): numpy's randn(1, N, 3) for every row, scaled, clipped and added on the device, kept within 50 m
    (lb2_jitter_filter);
  * the ground truth (:81-84): the first row of every 0.1 m voxel in row order, kept within 50 m (lb2_voxel_first_f64);
  * both shuffled by torch.randperm from torch's global CPU generator (the ground truth first), repeated element-wise and truncated
    to 2 num_points and num_points rows; mean and (unbiased) std of the ground truth (collations.py:20-39).

Seeded numpy / torch generators give the reference's samples: the same rows in the same order (DESIGN.md §3, refinement samples).
There is no CPU fallback: the dataset raises without the CUDA library or an sm_90 device.

    ds = TemporalKITTISet("Datasets/SemanticKITTI", 40, ["08"], "validation", 0.05, 180000, "refine")
    p_full, mean, std, p_noise, window = ds[0]
"""
from __future__ import annotations

import os

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from . import _lib, rng
from .datasets import SparseSegmentCollation, augment, repeat_rows
from .kitti import label_path, load_poses, read_labels, read_scan

NOISE_SIGMA, NOISE_CLIP = 0.2, 0.3      # SemanticKITTITemporalAggr.py:79
MAX_RANGE = 50.0                        # :90-91
DEDUP_VOXEL = 0.1                       # :81

SEGMENT_DTYPE = np.dtype([("start", "<i8"), ("m", "<f8", (12,))])     # lb2_segment


def window_list(names, scan_window):
    """the windows of one sequence's sorted scan names (:47-53): names[i : i + W] while more than 1.5 W names are left from i, then
    the rest as one last (longer) window"""
    out = []
    for i in range(len(names)):
        end = i + scan_window if len(names) - i > 1.5 * scan_window else len(names)
        out.append(names[i:end])
        if end == len(names):
            break
    return out


def repeat_to(rows: torch.Tensor, perm: torch.Tensor, n: int) -> torch.Tensor:
    """rows[perm].repeat(ceil(n / len), 0)[:n] with numpy's element-wise repeat (collations.py:32-36)"""
    times = int(np.ceil(n / rows.shape[0]))
    return repeat_rows(rows[perm.to(rows.device)], times)[:n]


class TemporalKITTISet(Dataset):
    def __init__(self, data_dir, scan_window, seqs, split, resolution, num_points, mode, device="cuda", device_rng=False):
        super().__init__()
        self.data_dir = data_dir
        self.n_clusters = 50
        self.resolution = resolution
        self.scan_window = scan_window
        self.num_points = num_points
        self.split = split
        self.seqs = seqs
        self.mode = mode
        self.device_rng = device_rng          # numpy's randn and torch's randperms drawn on the GPU (lidiff_b200.rng), the same values
        self.h = _lib.get_handle(device)
        self.device = self.h.device
        self.datapath_list()
        self.nr_data = len(self.points_datapath)
        print("The size of %s data is %d" % (self.split, len(self.points_datapath)))

    def datapath_list(self):
        """the windows of every sequence, and each sequence's poses, loaded once"""
        self.points_datapath = []
        self.seq_poses = {}
        for seq in self.seqs:
            seq_dir = os.path.join(self.data_dir, "dataset", "sequences", seq)
            names = sorted(os.listdir(os.path.join(seq_dir, "velodyne")))      # a plain sort, as :46
            self.seq_poses[seq] = load_poses(os.path.join(seq_dir, "calib.txt"), os.path.join(seq_dir, "poses.txt"))
            for w in window_list(names, self.scan_window):
                self.points_datapath.append([os.path.join(seq_dir, "velodyne", name) for name in w])

    def __len__(self):
        return self.nr_data

    # ---- the steps of __getitem__ -------------------------------------------------------------------------------------------
    def _pose(self, window, path):
        poses = self.seq_poses[path.split("/")[-3]]
        stem = os.path.basename(path).split(".")[0]
        try:
            k = int(stem)
        except ValueError:
            raise ValueError(f"window {window[0]} .. {window[-1]}: scan {path} has no integer stem (its pose index)") from None
        if not 0 <= k < len(poses):
            raise ValueError(f"window {window[0]} .. {window[-1]}: scan {path} has no pose (poses.txt has {len(poses)})")
        return poses[k]

    def aggregate(self, index: int) -> torch.Tensor:
        """[pcd_full; pcd_part] of aggregate_pcds as fp64 device rows: the scans other than t_frame in order, then t_frame"""
        window = self.points_datapath[index]
        t_frame = len(window) // 2
        order = [k for k in range(len(window)) if k != t_frame] + [t_frame]
        scans, labels = [], []
        seg = np.zeros(len(window), SEGMENT_DTYPE)
        start = 0
        for j, k in enumerate(order):
            path = window[k]
            pose = self._pose(window, path)
            scan = read_scan(path)
            lp = label_path(path)
            if not os.path.exists(lp):
                raise ValueError(f"window {window[0]} .. {window[-1]}: label file {lp} not found")
            labels.append(read_labels(lp, scan.shape[0]))
            scans.append(scan)
            seg[j]["start"] = start
            seg[j]["m"] = np.asarray(pose, dtype=np.float64)[:3, :4].reshape(-1)
            start += scan.shape[0]
        undo = np.linalg.inv(self._pose(window, window[-1]))           # the window's last scan, :124-126
        n, split = start, int(seg[-1]["start"])
        pts = torch.from_numpy(np.concatenate(scans)).to(self.device)
        lab = torch.from_numpy(np.concatenate(labels).view(np.int32)).to(self.device)
        d_seg = torch.from_numpy(seg.view(np.uint8)).to(self.device)
        out = torch.empty((max(n, 1), 3), dtype=torch.float64, device=self.device)
        d_out = torch.zeros(2, dtype=torch.int32, device=self.device)
        self.h.aggregate_window(pts, lab, d_seg, len(window), undo[:3, :4].reshape(-1), split, out, d_out,
                                self.h.aggregate_window_scratch(n))
        m, n_full = d_out.tolist()
        if m == n_full:
            raise ValueError(f"window {window[0]} .. {window[-1]}: no point of the frame scan {window[t_frame]} passes the "
                             "label / range filter")
        return out[:m]

    def __getitem__(self, index):
        window = self.points_datapath[index]
        p_concat = self.aggregate(index)
        if self.split == "train":
            p_concat = augment(p_concat)
        n = p_concat.shape[0]
        if self.device_rng:                                                     # numpy's global generator, every row
            r = rng.numpy_randn(1, n, 3, device=self.device)[0]
        else:
            r = torch.from_numpy(np.random.randn(1, n, 3)[0]).to(self.device)
        noise = torch.empty((n, 3), dtype=torch.float64, device=self.device)
        full = torch.empty((n, 3), dtype=torch.float64, device=self.device)
        counts = torch.zeros(3, dtype=torch.int32, device=self.device)
        self.h.jitter_filter(p_concat, r, NOISE_SIGMA, NOISE_CLIP, MAX_RANGE, noise, counts[0:1], self.h.jitter_filter_scratch(n))
        self.h.voxel_first_f64(p_concat, DEDUP_VOXEL, MAX_RANGE, full, counts[1:3], self.h.voxel_first_f64_scratch(n))
        n_noise, n_full, status = counts.tolist()
        where = f"window {window[0]} .. {window[-1]}"
        if status & 1:
            raise ValueError(f"{where}: a point's {DEDUP_VOXEL:g} m voxel index is outside +-2^20")
        if n_full == 0 or n_noise == 0:
            raise ValueError(f"{where}: no {'ground-truth' if n_full == 0 else 'noisy'} point lies within {MAX_RANGE:g} m")
        randperm = (lambda k: rng.torch_randperm(k, device=self.device)) if self.device_rng else torch.randperm
        perm_full = randperm(n_full)                             # torch's global CPU generator, collations.py:31, :34
        perm_noise = randperm(n_noise)
        p_full = repeat_to(full[:n_full], perm_full, 2 * self.num_points)
        p_noise = repeat_to(noise[:n_noise], perm_noise, self.num_points)
        return [p_full, p_full.mean(0), p_full.std(0), p_noise, window]

    def batch(self, indices) -> dict:
        """SparseSegmentCollation('refine') of the samples `indices`"""
        return SparseSegmentCollation("refine")([self[int(i)] for i in indices])


class TemporalKittiDataModule:
    """The reference's data module: its splits, batch sizes and shuffle flags, including the test loader over the TRAIN sequences
    (datasets_refine.py:58-71).  The loaders yield batches in the main process (the samples are built on the GPU, which worker
    processes cannot share), so the configured num_workers is not used."""

    def __init__(self, cfg, device="cuda", device_rng=None):
        self.cfg = cfg
        self.device = device
        # numpy's randn and torch's randperms drawn on the GPU (lidiff_b200.rng), the same values; None: the config's data.device_rng (default off)
        self.device_rng = bool(cfg["data"].get("device_rng", False)) if device_rng is None else bool(device_rng)

    def prepare_data(self):
        pass

    def setup(self, stage=None):
        pass

    def _loader(self, seqs, split, mode, batch_size, shuffle=False):
        d = self.cfg["data"]
        ds = TemporalKITTISet(data_dir=d["data_dir"], scan_window=d["scan_window"], seqs=seqs, split=split, resolution=d["resolution"],
                              num_points=d["num_points"], mode=mode, device=self.device,
                              device_rng=self.device_rng)
        return DataLoader(ds, batch_size=batch_size, shuffle=shuffle, num_workers=0, collate_fn=SparseSegmentCollation("refine"))

    def train_dataloader(self):
        return self._loader(self.cfg["data"]["train"], self.cfg["data"]["split"], "refine", self.cfg["train"]["batch_size"], True)

    def val_dataloader(self, pre_training=True):
        return self._loader(self.cfg["data"]["validation"], "validation", "refine", 1)

    def test_dataloader(self):
        return self._loader(self.cfg["data"]["train"], "validation", self.cfg["train"]["mode"], 1)


dataloaders = {"KITTI": TemporalKittiDataModule}
