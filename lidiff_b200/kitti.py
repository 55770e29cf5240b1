"""SemanticKITTI sequence files: calib.txt, poses.txt, velodyne/*.bin scans and labels/*.label files (the layout
lidiff/map_from_scans.py, lidiff/utils/eval_path.py and the reference's dataloader read)."""
from __future__ import annotations

import os
import re

import numpy as np


def _rows_4x4(values):
    pose = np.zeros((4, 4))
    pose[0, :4], pose[1, :4], pose[2, :4] = values[0:4], values[4:8], values[8:12]
    pose[3, 3] = 1.0
    return pose


def parse_calibration(filename: str) -> dict:
    """KITTI calib.txt: `KEY: 12 numbers` per line -> {KEY: 4x4}"""
    calib = {}
    with open(filename) as f:
        for line in f:
            if not line.strip():
                continue
            key, content = line.strip().split(":")
            calib[key] = _rows_4x4([float(v) for v in content.split()])
    return calib


def load_poses(calib_fname: str, poses_fname: str) -> list:
    """poses.txt (12 numbers per line) in the LiDAR frame: Tr^-1 . pose . Tr when calib.txt exists"""
    tr = parse_calibration(calib_fname)["Tr"] if os.path.exists(calib_fname) else None
    poses = []
    with open(poses_fname) as f:
        for line in f:
            if not line.strip():
                continue
            pose = _rows_4x4([float(v) for v in line.split()])
            poses.append(np.linalg.inv(tr) @ (pose @ tr) if tr is not None else pose)
    return poses


def natural_sorted(names):
    return sorted(names, key=lambda s: [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", s)])


def _read_into(path: str, out: np.ndarray, nbytes: int) -> None:
    view = memoryview(out.reshape(-1).view(np.uint8))[:nbytes]
    with open(path, "rb", buffering=0) as f:
        got = 0
        while got < nbytes:
            k = f.readinto(view[got:])
            if not k:
                raise OSError(f"{path}: short read ({got} of {nbytes} bytes)")
            got += k


def read_scan(path: str, out: np.ndarray | None = None) -> np.ndarray:
    """velodyne .bin -> (n, 4) float32 rows x, y, z, remission; read into the front of `out` (any dtype, enough bytes) when given"""
    nbytes = os.path.getsize(path)
    if nbytes % 16:
        raise ValueError(f"{path}: {nbytes} bytes is not a whole number of (x, y, z, remission) float32 rows")
    if out is None:
        return np.fromfile(path, dtype=np.float32).reshape(-1, 4)
    if out.nbytes < nbytes:
        raise ValueError(f"{path}: buffer of {out.nbytes} bytes is too small for {nbytes}")
    _read_into(path, out, nbytes)
    return out.reshape(-1).view(np.uint8)[:nbytes].view(np.float32).reshape(-1, 4)


def label_path(scan_path: str) -> str:
    """<seq>/velodyne/<stem>.bin -> <seq>/labels/<stem>.label"""
    seq = os.path.dirname(os.path.dirname(scan_path))
    return os.path.join(seq, "labels", os.path.splitext(os.path.basename(scan_path))[0] + ".label")


def read_labels(path: str, n: int | None = None, out: np.ndarray | None = None) -> np.ndarray:
    """.label -> uint32 (n,) (semantic class in the low 16 bits, instance id above); n = the scan's point count, checked"""
    if not os.path.exists(path):
        raise FileNotFoundError(f"label file not found: {path}")
    nbytes = os.path.getsize(path)
    if nbytes % 4 or (n is not None and nbytes != 4 * n):
        raise ValueError(f"{path}: {nbytes} bytes of labels" + (f" for a scan of {n} points" if n is not None else ""))
    if out is None:
        return np.fromfile(path, dtype=np.uint32)
    if out.nbytes < nbytes:
        raise ValueError(f"{path}: buffer of {out.nbytes} bytes is too small for {nbytes}")
    _read_into(path, out, nbytes)
    return out.reshape(-1).view(np.uint8)[:nbytes].view(np.uint32)
