"""A numpy restatement of the SemanticKITTI scene-completion grid format (lidiff_b200/ssc.py, include/lidiff_b200.h) and of what
csrc/ssc.cu computes from it: packed bits, occupancy, voxel centres, voxelization and the completion counts."""
import numpy as np

DIMS = (256, 256, 32)
N_VOXELS = 256 * 256 * 32
N_WORDS = N_VOXELS // 32
GRID_MIN = np.array([0.0, -25.6, -2.0])
VOXEL = 0.2


def unpack(words) -> np.ndarray:
    """bool (N_VOXELS,) of packed bits (uint32 words whose little-endian bytes are the file's, MSB first)"""
    return np.unpackbits(np.ascontiguousarray(words).view(np.uint8)).astype(bool)


def pack(occ) -> np.ndarray:
    """uint32 (N_WORDS,) words of a bool (N_VOXELS,) occupancy"""
    return np.packbits(np.asarray(occ, bool).reshape(-1)).view("<u4").copy()


def occupied(labels) -> np.ndarray:
    labels = np.asarray(labels)
    return (labels != 0) & (labels != 255)


def centres(occ) -> np.ndarray:
    """fp64 (P, 3) centres of the set voxels in ascending index order"""
    idx = np.stack(np.unravel_index(np.nonzero(np.asarray(occ).reshape(-1))[0], DIMS), 1)
    return GRID_MIN + (idx + 0.5) * VOXEL


def voxel_index(points):
    """(v int64 (n,) with -1 for dropped rows, non-finite mask, outside mask)"""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    finite = np.isfinite(p).all(1)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor((p - GRID_MIN) / VOXEL)
        inside = finite & ((f >= 0) & (f < np.array(DIMS))).all(1)
    v = np.full(p.shape[0], -1, np.int64)
    fi = f[inside].astype(np.int64)
    v[inside] = (fi[:, 0] * DIMS[1] + fi[:, 1]) * DIMS[2] + fi[:, 2]
    return v, ~finite, finite & ~inside


def voxelize(points):
    """(words uint32 (N_WORDS,), rows dropped as non-finite, rows dropped as outside)"""
    v, nf, out = voxel_index(points)
    occ = np.zeros(N_VOXELS, bool)
    occ[v[v >= 0]] = True
    return pack(occ), int(nf.sum()), int(out.sum())


def confusion(pred_words, gt_labels, invalid_words=None):
    """(TP, FP, FN) over the valid voxels: label != 255 and not set in .invalid"""
    pred = unpack(pred_words)
    labels = np.asarray(gt_labels)
    valid = labels != 255
    if invalid_words is not None:
        valid &= ~unpack(invalid_words)
    gt = occupied(labels) & valid
    return int((pred & gt).sum()), int((pred & ~gt & valid).sum()), int((~pred & gt).sum())


def random_labels(rng, density, ignore=0.0):
    """uint16 labels: occupied with probability `density` (classes 1..254 and 256..259), 255 with probability `ignore`"""
    u = rng.random(N_VOXELS)
    lab = np.where(u < density, rng.choice(np.r_[1:255, 256:260], N_VOXELS), 0).astype(np.uint16)
    lab[(u >= density) & (u < density + ignore)] = 255
    return lab
