"""The diffusion network's SemanticKITTI samples on the GPU — the reference's `TemporalKITTISet`
(lidiff/datasets/dataloader/SemanticKITTITemporal.py), `point_set_to_sparse` / `SparseSegmentCollation` (lidiff/utils/collations.py)
and `TemporalKittiDataModule` (lidiff/datasets/datasets.py).

Per sample, as the reference's __getitem__ (line numbers of SemanticKITTITemporal.py / collations.py):
  * the scan's label, range and height filter (:82-94) and the crop of the sequence map about the scan pose, transformed into the
    scan frame (:99-105): one lb2_select_points call each; the maps stay resident on the device;
  * the training augmentation (:69-76, utils/pcd_transforms.py) with its random numbers drawn on the host from numpy's global
    generator in the reference's order, applied to the rows on the device;
  * the partial scan repeated element-wise and sampled by farthest point sampling (collations.py:42-48);
  * the 10 m viewpoint grid of the partial scan and the map points it includes (:46, :50-51: lb2_viewpoint_filter), shuffled by a
    torch.randperm drawn from torch's global CPU generator, repeated element-wise and truncated (:52-57);
  * mean and (unbiased) std over the rows, or the dataset statistics of utils/data_stats_range_<r>m.yml (:60-61).

Seeded numpy / torch generators give the reference's samples: the same rows in the same order (DESIGN.md §3, training samples).
There is no CPU fallback: the dataset raises without the CUDA library or an sm_90 device.

    ds = TemporalKITTISet("Datasets/SemanticKITTI", ["08"], "validation", 0.05, 180000, 50.0)
    p_full, mean, std, p_part, filename = ds[0]
    batch = ds.batch([0, 1])            # SparseSegmentCollation's dict; the partial scans' FPS in one launch from 3 scans on
"""
from __future__ import annotations

import os

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from . import _lib, rng
from .kitti import label_path, load_poses, natural_sorted, read_labels, read_scan
from .pipeline import FPS_CLUSTER_MIN_SCANS
from .preprocess import farthest_point_sample, farthest_point_sample_batched

VIEWPOINT_VOXEL = 10.0          # collations.py:46
MIN_RANGE = 3.5                 # SemanticKITTITemporal.py:93
MIN_Z = -4.0                    # :94, :105


def _desc(range_mode=_lib.RANGE_NONE, center=(0.0, 0.0, 0.0), r_min=-np.inf, r_max=np.inf, transform=None, z_min=None):
    d = _lib.SelectDesc()
    d.range_mode = range_mode
    d.center[:] = [float(v) for v in center]
    d.r_min, d.r_max = float(r_min), float(r_max)
    d.has_transform = int(transform is not None)
    if transform is not None:
        d.transform[:] = [float(v) for v in np.asarray(transform, dtype=np.float64)[:3, :4].reshape(-1)]
    d.has_z_min = int(z_min is not None)
    d.z_min = float(z_min) if z_min is not None else 0.0
    return d


def _rotate_f32(p: torch.Tensor, R: np.ndarray) -> torch.Tensor:
    """np.dot(p, R) in fp64 stored into a float32 array (pcd_transforms.py:13, :32), read back as fp64"""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    cols = [(x * float(R[0, k]) + y * float(R[1, k])) + z * float(R[2, k]) for k in range(3)]
    return torch.stack(cols, 1).float().double()


def augment(p: torch.Tensor) -> torch.Tensor:
    """TemporalKITTISet.transforms (:69-76) on fp64 rows: rotate_point_cloud, rotate_perturbation_point_cloud, random_scale_point_cloud,
    random_flip_point_cloud; the random numbers come from numpy's global generator in the reference's order"""
    angle = np.random.uniform() * 2 * np.pi
    c, s = np.cos(angle), np.sin(angle)
    p = _rotate_f32(p, np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]))
    a = np.clip(0.06 * np.random.randn(3), -0.18, 0.18)
    Rx = np.array([[1, 0, 0], [0, np.cos(a[0]), -np.sin(a[0])], [0, np.sin(a[0]), np.cos(a[0])]])
    Ry = np.array([[np.cos(a[1]), 0, np.sin(a[1])], [0, 1, 0], [-np.sin(a[1]), 0, np.cos(a[1])]])
    Rz = np.array([[np.cos(a[2]), -np.sin(a[2]), 0], [np.sin(a[2]), np.cos(a[2]), 0], [0, 0, 1]])
    p = _rotate_f32(p, np.dot(Rz, np.dot(Ry, Rx)))
    p = p * float(np.random.uniform(0.95, 1.05, 1)[0])
    if np.random.random() > 0.5:
        p[:, 1] = -p[:, 1]
    return p


def repeat_rows(p: torch.Tensor, times: int) -> torch.Tensor:
    """numpy's p.repeat(times, 0): every row `times` times in a row ([a, a, b, b, ...]), not tiling"""
    return p.repeat_interleave(int(times), dim=0)


class TemporalKITTISet(Dataset):
    def __init__(self, data_dir, seqs, split, resolution, num_points, max_range, dataset_norm=False, std_axis_norm=False,
                 device="cuda", device_rng=False):
        super().__init__()
        self.data_dir = data_dir
        self.n_clusters = 50
        self.resolution = resolution
        self.num_points = num_points
        self.max_range = max_range
        self.split = split
        self.seqs = seqs
        self.device_rng = device_rng          # the map crop's torch randperm drawn on the GPU (lidiff_b200.rng), the same values
        self.h = _lib.get_handle(device)
        self.device = self.h.device
        self.cache_maps = {}
        self.datapath_list()
        self.data_stats = {"mean": None, "std": None}
        stats_file = f"utils/data_stats_range_{int(self.max_range)}m.yml"
        if os.path.isfile(stats_file) and dataset_norm:
            import yaml
            with open(stats_file) as f:
                stats = yaml.safe_load(f)
            data_mean = np.array([stats["mean_axis"]["x"], stats["mean_axis"]["y"], stats["mean_axis"]["z"]])
            if std_axis_norm:
                data_std = np.array([stats["std_axis"]["x"], stats["std_axis"]["y"], stats["std_axis"]["z"]])
            else:
                data_std = np.array([stats["std"], stats["std"], stats["std"]])
            self.data_stats = {"mean": torch.tensor(data_mean), "std": torch.tensor(data_std)}
        self.nr_data = len(self.points_datapath)
        print("The size of %s data is %d" % (self.split, len(self.points_datapath)))

    def datapath_list(self):
        """scan paths and poses of every sequence; the sequence maps are uploaded once (the reference's cache_maps), none for 'test'"""
        self.points_datapath = []
        self.seq_poses = []
        for seq in self.seqs:
            seq_dir = os.path.join(self.data_dir, "dataset", "sequences", seq)
            names = natural_sorted(os.listdir(os.path.join(seq_dir, "velodyne")))
            poses = load_poses(os.path.join(seq_dir, "calib.txt"), os.path.join(seq_dir, "poses.txt"))
            if self.split != "test":
                m = np.load(os.path.join(seq_dir, "map_clean.npy"))
                if m.ndim != 2 or m.shape[1] not in (3, 4):
                    raise ValueError(f"{seq_dir}/map_clean.npy: expected (n, 3) points, got shape {m.shape}")
                if m.dtype not in (np.float32, np.float64):
                    m = m.astype(np.float64)
                self.cache_maps[seq] = torch.from_numpy(np.ascontiguousarray(m)).to(self.device)
            else:
                self.cache_maps[seq] = None
            for k, name in enumerate(names):
                self.points_datapath.append(os.path.join(seq_dir, "velodyne", name))
                self.seq_poses.append(poses[k])

    def __len__(self):
        return self.nr_data

    # ---- the steps of __getitem__ -------------------------------------------------------------------------------------------
    def _select(self, points: torch.Tensor, labels, desc, out: torch.Tensor, d_count: torch.Tensor):
        scratch = self.h.select_points_scratch(points.shape[0])
        self.h.select_points(points, labels, desc, out, d_count, scratch)

    def _filtered(self, index: int):
        """(partial scan, cropped map or None) as fp64 device rows after the filters of :82-105"""
        path = self.points_datapath[index]
        scan = torch.from_numpy(read_scan(path)).to(self.device)
        labels = None
        if self.split != "test":
            labels = torch.from_numpy(read_labels(label_path(path), scan.shape[0]).view(np.int32)).to(self.device)
        counts = torch.zeros(2, dtype=torch.int32, device=self.device)
        part = torch.empty((scan.shape[0], 3), dtype=torch.float64, device=self.device)
        self._select(scan, labels, _desc(_lib.RANGE_FP32, r_min=MIN_RANGE, r_max=self.max_range, z_min=MIN_Z), part, counts[0:1])
        full = None
        if self.split != "test":
            pose = self.seq_poses[index]
            p_map = self.cache_maps[path.split("/")[-3]]
            full = torch.empty((p_map.shape[0], 3), dtype=torch.float64, device=self.device)
            self._select(p_map, None, _desc(_lib.RANGE_FP64, center=pose[:-1, -1], r_max=self.max_range, transform=np.linalg.inv(pose),
                                            z_min=MIN_Z), full, counts[1:2])
        n_part, n_full = counts.tolist()
        return part[:n_part], (full[:n_full] if full is not None else None)

    def _prepare(self, index: int):
        """everything of __getitem__ but the farthest point sampling, which has no random draws:
        (repeated partial scan, p_full, mean, std, filename)"""
        path = self.points_datapath[index]
        p_part, p_full = self._filtered(index)
        if p_part.shape[0] == 0:
            raise ValueError(f"{path}: no point of the scan passes the label / range / height filter")
        test = p_full is None
        if test:
            p_full = p_part
        if self.split == "train":
            cat = augment(torch.cat([p_full, p_part]))
            p_full, p_part = cat[: -p_part.shape[0]], cat[-p_part.shape[0]:]
        n_part = int(self.num_points / 10.0)
        part_rep = repeat_rows(p_part, np.ceil(n_part / p_part.shape[0]))
        inc = torch.empty_like(p_full)
        d_out = torch.zeros(2, dtype=torch.int32, device=self.device)
        scratch = self.h.viewpoint_filter_scratch(p_part.shape[0], p_full.shape[0])
        self.h.viewpoint_filter(p_part.contiguous(), p_full.contiguous(), VIEWPOINT_VOXEL, inc, d_out, scratch)
        n_in, status = d_out.tolist()
        if status & 1:
            raise ValueError(f"{path}: the partial scan spans more than 2^21 viewpoint cells along an axis")
        if n_in == 0:
            raise ValueError(f"{path}: no point of the ground-truth map lies in the partial scan's {VIEWPOINT_VOXEL:g} m viewpoint grid")
        # torch's global CPU generator, as collations.py:54
        perm = rng.torch_randperm(n_in, device=self.device) if self.device_rng else torch.randperm(n_in)
        times = int(np.ceil(self.num_points / n_in))
        rows = perm.to(self.device)[torch.arange(self.num_points, device=self.device) // times]
        p_full = inc[:n_in][rows]
        if test:                                                  # the reference's p_full is the float32 scan here
            mean = p_full.mean(0).float() if self.data_stats["mean"] is None else self.data_stats["mean"]
            std = p_full.std(0).float() if self.data_stats["std"] is None else self.data_stats["std"]
            p_full = p_full.float()
        else:
            mean = p_full.mean(0) if self.data_stats["mean"] is None else self.data_stats["mean"]
            std = p_full.std(0) if self.data_stats["std"] is None else self.data_stats["std"]
        return part_rep, p_full, mean, std, path

    def __getitems__(self, indices):
        """[self[i] for i in indices], the partial scans' farthest point sampling in one launch when there are at least
        FPS_CLUSTER_MIN_SCANS of them (the same indices either way)"""
        prepared = [self._prepare(int(i)) for i in indices]
        n_part = int(self.num_points / 10.0)
        reps = [p[0] for p in prepared]
        if len(reps) >= FPS_CLUSTER_MIN_SCANS:
            sel = farthest_point_sample_batched(reps, n_part)
        else:
            sel = [farthest_point_sample(r, n_part) for r in reps]
        return [[p_full, mean, std, rep[s], path] for (rep, p_full, mean, std, path), s in zip(prepared, sel)]

    def __getitem__(self, index):
        return self.__getitems__([index])[0]

    def batch(self, indices) -> dict:
        """SparseSegmentCollation of the samples `indices`"""
        return SparseSegmentCollation()(self.__getitems__(indices))


class SparseSegmentCollation:
    def __init__(self, mode="diffusion"):
        self.mode = mode

    def __call__(self, data):
        batch = list(zip(*data))
        return {"pcd_full": torch.stack(batch[0]).float(),
                "mean": torch.stack(batch[1]).float(),
                "std": torch.stack(batch[2]).float(),
                "pcd_part" if self.mode == "diffusion" else "pcd_noise": torch.stack(batch[3]).float(),
                "filename": batch[4]}


class TemporalKittiDataModule:
    """The reference's data module: its splits, batch sizes and shuffle flags.  The loaders yield batches in the main process
    (the samples are built on the GPU, which worker processes cannot share), so the configured num_workers is not used."""

    def __init__(self, cfg, device="cuda", device_rng=None):
        self.cfg = cfg
        self.device = device
        # the map crop's torch randperm drawn on the GPU (lidiff_b200.rng), the same values; None: the config's data.device_rng (default off)
        self.device_rng = bool(cfg["data"].get("device_rng", False)) if device_rng is None else bool(device_rng)

    def prepare_data(self):
        pass

    def setup(self, stage=None):
        pass

    def _set(self, seqs, split):
        d = self.cfg["data"]
        return TemporalKITTISet(data_dir=d["data_dir"], seqs=seqs, split=split, resolution=d["resolution"], num_points=d["num_points"],
                                max_range=d["max_range"], dataset_norm=d["dataset_norm"], std_axis_norm=d["std_axis_norm"],
                                device=self.device, device_rng=self.device_rng)

    def train_dataloader(self):
        return DataLoader(self._set(self.cfg["data"]["train"], self.cfg["data"]["split"]), batch_size=self.cfg["train"]["batch_size"],
                          shuffle=True, num_workers=0, collate_fn=SparseSegmentCollation())

    def val_dataloader(self, pre_training=True):
        return DataLoader(self._set(self.cfg["data"]["validation"], "validation"), batch_size=1, num_workers=0,
                          collate_fn=SparseSegmentCollation())

    def test_dataloader(self):
        return DataLoader(self._set(self.cfg["data"]["validation"], "validation"), batch_size=self.cfg["train"]["batch_size"],
                          num_workers=0, collate_fn=SparseSegmentCollation())


dataloaders = {"KITTI": TemporalKittiDataModule}
