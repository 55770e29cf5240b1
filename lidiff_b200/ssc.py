"""SemanticKITTI scene-completion (SSC) voxel grids on the GPU: read and write the dataset's grid files, turn grids into points and
points into grids, and count the benchmark's scene-completion IoU, precision and recall.

The format, restated from the SemanticKITTI development kit (semantic-kitti-api: auxiliary/io_data.py's `unpack` and the extents
of generate_sequential.py), and pinned in one place here and in include/lidiff_b200.h:

  * The grid is DIMS = (256, 256, 32) voxels of VOXEL_SIZE = 0.2 m in C order, v = (i 256 + j) 32 + k, over [GRID_MIN, GRID_MAX)
    with GRID_MIN = (0, -25.6, -2) and GRID_MAX = (51.2, 25.6, 4.4), in the scan's frame.
  * `.bin` / `.invalid`: BIN_BYTES = 262 144 bytes, voxel v is bit 7 - (v & 7) of byte v >> 3 (MSB first, np.unpackbits' default
    order).  In memory a packed grid is N_WORDS uint32 whose little-endian bytes are the file's bytes.
  * `.label`: N_VOXELS little-endian uint16; 0 = empty, IGNORE = 255.  A voxel is occupied iff its label is neither.  In the
    dataset's ground truth, voxels set in `.invalid` count as IGNORE.
  * Voxel -> point: the centre, GRID_MIN_d + (idx_d + 0.5) 0.2 in fp64 (product and sum each rounded); points come out in
    ascending v (np.nonzero's order).
  * Point -> voxel: idx_d = floor((p_d - GRID_MIN_d) / 0.2) in fp64; a point is kept iff every index is in range.  A point with a
    NaN / inf coordinate is dropped and counted, never clamped.

A file of the wrong size raises ValueError naming the file and its size.  Occupancy only: the semantic classes of the labels and
the benchmark's per-class mIoU are not used.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib

DIMS = (256, 256, 32)
N_VOXELS = 256 * 256 * 32
N_WORDS = N_VOXELS // 32
BIN_BYTES = N_VOXELS // 8
LABEL_BYTES = 2 * N_VOXELS
VOXEL_SIZE = 0.2
GRID_MIN = (0.0, -25.6, -2.0)
GRID_MAX = (51.2, 25.6, 4.4)
IGNORE = 255
KINDS = {"bits": _lib.SSC_BITS, "labels": _lib.SSC_LABELS}
CHUNK = 32                          # grids per grid_points launch group: 4 launches and one host read each


def _read(path: str, nbytes: int) -> bytes:
    size = os.path.getsize(path)
    if size != nbytes:
        raise ValueError(f"{path}: {size} bytes, an SSC grid file of this kind has {nbytes}")
    with open(path, "rb") as f:
        return f.read()


def read_grid(path: str) -> tuple[np.ndarray, str]:
    """(grid, kind) of a `.label` file (uint16 (N_VOXELS,), "labels") or a packed `.bin` / `.invalid` file (uint32 (N_WORDS,),
    "bits")"""
    if path.endswith(".label"):
        return np.frombuffer(_read(path, LABEL_BYTES), "<u2").copy(), "labels"
    if path.endswith((".bin", ".invalid")):
        return read_invalid(path), "bits"
    raise ValueError(f"{path}: an SSC grid is a .label, .bin or .invalid file")


def read_invalid(path: str) -> np.ndarray:
    """the packed bits of a `.invalid` (or `.bin`) file as uint32 (N_WORDS,)"""
    return np.frombuffer(_read(path, BIN_BYTES), "<u4").copy()


def write_bin(path: str, bits) -> None:
    """write packed bits (N_WORDS 32-bit words, numpy or torch, any device) as a `.bin` file"""
    b = bits.detach().cpu().numpy() if isinstance(bits, torch.Tensor) else np.asarray(bits)
    if b.size * b.itemsize != BIN_BYTES:
        raise ValueError(f"write_bin: {b.size * b.itemsize} bytes of bits, a grid has {BIN_BYTES}")
    with open(path, "wb") as f:
        f.write(np.ascontiguousarray(b).view(np.uint8).tobytes())


def _stack(grids, kind: str, device) -> torch.Tensor:
    """(G, N_VOXELS) uint16 labels or (G, N_WORDS) int32 words, contiguous on the device"""
    n, dt = (N_VOXELS, torch.int16) if kind == "labels" else (N_WORDS, torch.int32)
    if isinstance(grids, (list, tuple)):
        arrs = [g.detach().cpu().numpy() if isinstance(g, torch.Tensor) else np.asarray(g) for g in grids]
        grids = np.stack(arrs) if arrs and all(a.size == n for a in arrs) else np.zeros(0, np.uint8)
    t = grids.detach() if isinstance(grids, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(grids))
    if t.numel() == 0 or t.numel() % n or t.element_size() != torch.empty(0, dtype=dt).element_size():
        raise ValueError(f"expected {kind} grids of {n} {'uint16' if kind == 'labels' else 'uint32'} values each")
    t = t.reshape(-1, n)
    return t.view(dt).to(device=device).contiguous()


def grid_points(grids, kind: str, device="cuda") -> tuple[torch.Tensor, np.ndarray]:
    """(points fp64 (P, 3) on the device, offsets int64 (G + 1,)): the centres of the occupied voxels of G grids, grid after
    grid, each in ascending voxel order; grid g's rows are [offsets[g], offsets[g + 1]).  `grids`: one grid, a list of grids or a
    stacked (G, ...) array / tensor of `kind` "labels" (uint16) or "bits" (packed uint32 words).  CHUNK grids at a time: four
    launches and one host read each."""
    if kind not in KINDS:
        raise ValueError(f"kind must be one of {sorted(KINDS)}, got {kind!r}")
    h = _lib.get_handle(device)
    g = _stack(grids, kind, h.device)
    parts, offsets = [], [np.zeros(1, np.int64)]
    for c0 in range(0, g.shape[0], CHUNK):
        chunk = g[c0:c0 + CHUNK]
        off = torch.empty(chunk.shape[0] + 1, dtype=torch.int64, device=h.device)
        scratch = h.ssc_scratch(chunk.shape[0])
        h.ssc_grid_count(chunk, KINDS[kind], chunk.shape[0], off, scratch)
        off_h = off.cpu().numpy()                                           # the one host read: the chunk's point count
        out = torch.empty((int(off_h[-1]), 3), dtype=torch.float64, device=h.device)
        if out.shape[0]:
            h.ssc_grid_points(chunk.shape[0], off, scratch, out)
        parts.append(out)
        offsets.append(off_h[1:] + offsets[-1][-1])
    pts = parts[0] if len(parts) == 1 else torch.cat(parts)
    return pts, np.concatenate(offsets)


def voxelize(points, offsets=None, device="cuda") -> tuple[torch.Tensor, np.ndarray]:
    """(bits, dropped): the packed grid(s) of fp64 points and the rows dropped, (non-finite, outside the grid).  One cloud (n, 3):
    bits int32 (N_WORDS,) and dropped (2,); with `offsets` (G + 1 row bounds) G clouds: bits (G, N_WORDS) and dropped (G, 2)."""
    h = _lib.get_handle(device)
    p = points.detach() if isinstance(points, torch.Tensor) else torch.as_tensor(np.asarray(points, dtype=np.float64))
    if p.dim() != 2 or p.shape[1] != 3:
        raise ValueError(f"expected (n, 3) points, got {tuple(p.shape)}")
    p = p.to(device=h.device, dtype=torch.float64).contiguous()
    off = np.array([0, p.shape[0]], np.int64) if offsets is None else np.asarray(offsets, np.int64)
    if off.ndim != 1 or off.shape[0] < 2 or off[0] != 0 or off[-1] != p.shape[0] or (np.diff(off) < 0).any():
        raise ValueError(f"offsets must rise from 0 to the {p.shape[0]} rows")
    n_grids = off.shape[0] - 1
    bits = torch.empty((n_grids, N_WORDS), dtype=torch.int32, device=h.device)
    info = torch.empty(n_grids * C.sizeof(_lib.SscVoxelInfo), dtype=torch.uint8, device=h.device)
    h.ssc_voxelize(p, torch.from_numpy(off).to(h.device), n_grids, bits, info)
    dropped = info.cpu().numpy().view(np.int64).reshape(n_grids, 2).copy()
    return (bits[0], dropped[0]) if offsets is None else (bits, dropped)


def completion_counts(pred_bits, gt_labels, invalid=None, device="cuda") -> np.ndarray:
    """int64 (TP, FP, FN) of packed predicted occupancy against ground-truth labels (and packed `.invalid` bits, None: none) over
    the valid voxels; for one grid (3,), for stacked grids (G, 3)"""
    h = _lib.get_handle(device)
    single = np.asarray(gt_labels).ndim == 1 if not isinstance(gt_labels, torch.Tensor) else gt_labels.dim() == 1
    lab = _stack(gt_labels, "labels", h.device)
    pred = _stack(pred_bits, "bits", h.device)
    inv = None if invalid is None else _stack(invalid, "bits", h.device)
    if pred.shape[0] != lab.shape[0] or (inv is not None and inv.shape[0] != lab.shape[0]):
        raise ValueError("completion_counts: the predictions, labels and invalid masks must hold the same number of grids")
    out = torch.empty((lab.shape[0], 3), dtype=torch.int64, device=h.device)
    h.ssc_confusion(pred, lab, inv, lab.shape[0], out)
    res = out.cpu().numpy()
    return res[0] if single else res


class SSCCompletion:
    """the SSC benchmark's scene-completion scores, occupancy only: TP / FP / FN summed over scans, then
    IoU = TP / (TP + FP + FN), precision = TP / (TP + FP) and recall = TP / (TP + FN).  Restated from the development kit's
    evaluate_completion.py as remembered (its confusion matrix over the valid voxels; precision and recall with its 1e-8 guard),
    not verified against it.  A score whose denominator is 0 is nan (IoU) or 0 (precision, recall)."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.tp = self.fp = self.fn = 0
        self.scans = 0

    def add(self, counts):
        tp, fp, fn = (int(c) for c in counts)
        self.tp += tp
        self.fp += fp
        self.fn += fn
        self.scans += 1

    def compute(self) -> dict:
        tp, fp, fn = float(self.tp), float(self.fp), float(self.fn)
        return {"iou": tp / (tp + fp + fn) if tp + fp + fn else float("nan"),
                "precision": tp / (tp + fp + 1e-8), "recall": tp / (tp + fn + 1e-8)}
