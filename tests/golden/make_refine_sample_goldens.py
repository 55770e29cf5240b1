"""Records the samples the reference's refinement `TemporalKITTISet` (lidiff/datasets/dataloader/SemanticKITTITemporalAggr.py) builds
on a seeded synthetic SemanticKITTI layout, so lidiff_b200.datasets_refine can be compared against them without the reference's
source tree:

    python tests/golden/make_refine_sample_goldens.py REF   # REF = a checkout of the reference -> tests/golden/refine_samples_reference.npz

The reference's class runs unchanged on the shims, with three stand-ins: `hdbscan` and `matplotlib` (imported by
utils/pcd_preprocess.py, never called here) are empty modules, and ME.utils.sparse_quantize is make_map_goldens'
flooring_sparse_quantize (floor, then the first occurrence of every voxel in ascending row order) instead of the shim's truncating
one.  The scans are make_sample_goldens' (excluded classes 252.. and kept classes 0, 1, .. 251 with instance bits, a NaN and an inf
row per scan, points near the 3.5 m and 50 m boundaries), written by its write_sequence with distinct poses per scan; the windows
of SCAN_WINDOW = 3 scans include the longer tail window of a sequence and a 1-scan sequence.

The 3.5 m decisions are kept GEN_MARGIN clear by the generator.  The decisions made on the sample's rows are checked instead: the
recording fails if a row of [pcd_full; pcd_part] or of the noisy rows lies within FACE_ULPS float32 ulps of 50 m, or an augmented
(train) row within that distance of a 0.1 m voxel face, so an augmentation whose rotation rounds differently by one float32 ulp
cannot change a decision.  Without augmentation the rows are fp64 results of a fixed operation order, equal bit for bit.
"""
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SEED = 5
SCAN_WINDOW = 3
NUM_POINTS = 800
RESOLUTION = 0.05
FACE_ULPS = 3
SEQUENCES = {"00": 7, "01": 1, "08": 4}                          # name -> scans
TRAIN, VALIDATION = ["00", "01"], ["08"]
RECORD = {"train": [0, 4], "validation": [0], "test": [3, 4]}    # indices recorded per split, in this order


def make_dataset(root, seed=None):
    """root/dataset/sequences/{00, 01, 08}: scans, labels, calib.txt and poses.txt (and a map file the refinement path never reads)"""
    from make_sample_goldens import write_sequence
    seed = SEED if seed is None else seed
    for i, (seq, n) in enumerate(SEQUENCES.items()):
        write_sequence(os.path.join(root, "dataset", "sequences", seq), n, seed * 100 + i)
    return root


def split_seqs(split):
    """the data module's sequences: the test loader runs over the training sequences"""
    return VALIDATION if split == "validation" else TRAIN


def split_name(split):
    return "train" if split == "train" else "validation"


def record_key(split, k, what):
    return f"{split}_{k}_{what}"


def _ulp_margin(v, edge):
    """how many float32 ulps of |v| the fp64 values v lie from `edge` (finite values only)"""
    v = np.asarray(v, dtype=np.float64)
    edge = np.broadcast_to(np.asarray(edge, dtype=np.float64), v.shape).ravel()
    v = v.ravel()
    fin = np.isfinite(v)
    v, edge = v[fin], edge[fin]
    if not len(v):
        return np.inf
    return (np.abs(v - edge) / np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)).min()


def main(ref):
    import importlib
    import torch
    import lidiff_b200.shims as sh
    from make_map_goldens import flooring_sparse_quantize
    sh.install()
    sys.modules.setdefault("hdbscan", types.ModuleType("hdbscan"))
    mpl = sys.modules.setdefault("matplotlib", types.ModuleType("matplotlib"))
    plt = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot = plt
    sys.modules["matplotlib.pyplot"] = plt
    import MinkowskiEngine as ME
    worst = {"face": np.inf, "range": np.inf}
    augmented = [False]

    def quantize_checked(coordinates, **kw):
        c = np.asarray(coordinates, dtype=np.float64)
        fin = np.isfinite(c).all(1)
        p = c[fin] * 0.1                                              # the row the quotient came from, to within an fp64 ulp
        q = c[fin]
        if augmented[0]:
            worst["face"] = min(worst["face"], _ulp_margin(p, np.round(q) * 0.1))
        worst["range"] = min(worst["range"], _ulp_margin(np.sqrt((p ** 2).sum(1)), 50.0))
        return flooring_sparse_quantize(coordinates, **kw)
    ME.utils.sparse_quantize = quantize_checked

    sys.path.insert(0, ref)
    for k in [k for k in sys.modules if k == "lidiff" or k.startswith("lidiff.")]:
        sys.modules.pop(k)
    mod = importlib.import_module("lidiff.datasets.dataloader.SemanticKITTITemporalAggr")
    jitter = mod.jitter_point_cloud

    def jitter_checked(batch_data, **kw):
        out = jitter(batch_data, **kw)
        worst["range"] = min(worst["range"], _ulp_margin(np.sqrt((out[0] ** 2).sum(-1)), 50.0))
        return out
    mod.jitter_point_cloud = jitter_checked

    out = {"seed": np.array(SEED), "num_points": np.array(NUM_POINTS), "scan_window": np.array(SCAN_WINDOW)}
    with tempfile.TemporaryDirectory() as root:
        make_dataset(root)
        for split, indices in RECORD.items():
            ds = mod.TemporalKITTISet(root, SCAN_WINDOW, split_seqs(split), split_name(split), RESOLUTION, NUM_POINTS, "refine")
            augmented[0] = split == "train"
            np.random.seed(SEED)
            torch.manual_seed(SEED)
            for k, i in enumerate(indices):
                p_full, mean, std, p_noise, window = ds[i]
                out[record_key(split, k, "index")] = np.array(i)
                out[record_key(split, k, "pcd_full")] = p_full.numpy()
                out[record_key(split, k, "mean")] = mean.numpy()
                out[record_key(split, k, "std")] = std.numpy()
                out[record_key(split, k, "pcd_noise")] = p_noise.numpy()
                out[record_key(split, k, "window")] = np.array(["/".join(p.split("/")[-3:]) for p in window])
    assert worst["face"] >= FACE_ULPS, f"a row lies {worst['face']:.3g} fp32 ulps from a voxel face: choose another SEED"
    assert worst["range"] >= FACE_ULPS, f"a row lies {worst['range']:.3g} fp32 ulps from 50 m: choose another SEED"
    np.savez_compressed(os.path.join(HERE, "refine_samples_reference.npz"), **out)
    print({k: v.shape for k, v in out.items() if v.ndim}, "closest face / range (fp32 ulps)", worst)


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
