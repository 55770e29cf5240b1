"""Host logic of lidiff_b200.datasets on the numpy stand-in backend (tests/fake_samples_backend.py): the reference's recorded samples
for the train, validation and test splits, the order of the random draws, numpy's element-wise repeat, batch() against collated
items, the test split without a map, the errors for empty samples and the data module's splits."""
import os
import shutil
import sys

import numpy as np
import pytest
import torch
from torch.utils.data import RandomSampler, SequentialSampler

import fake_samples_backend
from lidiff_b200 import datasets as D

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_sample_goldens as G  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "samples_reference.npz"))


@pytest.fixture(scope="module")
def data_root(tmp_path_factory):
    return G.make_dataset(str(tmp_path_factory.mktemp("kitti")))


@pytest.fixture
def fake(monkeypatch):
    return fake_samples_backend.install(monkeypatch)


def make_set(root, split, device="cpu"):
    return D.TemporalKITTISet(root, G.split_seqs(split), split, G.RESOLUTION, G.NUM_POINTS, G.MAX_RANGE, device=device)


def assert_close_to_golden(split, k, item):
    """rows in the same order: within 2 float32 ulps of the golden (1 ulp before the scale in [0.95, 1.05]) for the train split, 4
    fp64 ulps of the pose product's magnitude otherwise; mean / std within 1e-12 relative.  The test split's statistics are float32
    sums in the reference, whose rounding error scales with the summands, not with the result: within 1e-6 (|mean| + std) there"""
    p_full, mean, std, p_part, fname = item
    for name, got in (("pcd_full", p_full), ("pcd_part", p_part)):
        ref = GOLDEN[G.record_key(split, k, name)]
        got = got.cpu().numpy()
        assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape, got.dtype, ref.dtype)
        if split == "train":
            tol = 2 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
        else:       # 4 ulps of the sum the pose product forms: |x| + |y| + |z| of the row and the pose translation (< 4 m here)
            tol = 4 * np.spacing(np.abs(ref.astype(np.float64)).sum(1, keepdims=True) + 4.0)
        err = np.abs(got.astype(np.float64) - ref.astype(np.float64))
        assert (err <= tol).all(), (split, k, name, err.max())
    scale = np.abs(GOLDEN[G.record_key(split, k, "mean")]).astype(np.float64) + GOLDEN[G.record_key(split, k, "std")]
    for name, got in (("mean", mean), ("std", std)):
        ref = GOLDEN[G.record_key(split, k, name)]
        if split == "test":
            err = np.abs(got.cpu().numpy().astype(np.float64) - ref)
            assert (err <= 1e-6 * scale).all(), (split, k, name, err, scale)
        else:
            np.testing.assert_allclose(got.cpu().numpy(), ref, rtol=1e-12, atol=0, err_msg=f"{split} {k} {name}")
    assert "/".join(fname.split("/")[-3:]) == str(GOLDEN[G.record_key(split, k, "filename")])


@pytest.mark.parametrize("split", ["train", "validation", "test"])
def test_items_match_reference(fake, data_root, split):
    ds = make_set(data_root, split)
    np.random.seed(G.SEED)
    torch.manual_seed(G.SEED)
    for k, i in enumerate(G.RECORD[split]):
        assert int(GOLDEN[G.record_key(split, k, "index")]) == i
        assert_close_to_golden(split, k, ds[i])


def test_recorded_samples_cover_repeat_and_truncation(fake, data_root):
    """the recorded train and validation samples include partial scans shorter and longer than num_points / 10, and
    viewpoint-filtered maps shorter than num_points (repeated: fewer distinct rows) and longer (truncated: all rows distinct)"""
    n_part = int(G.NUM_POINTS / 10)
    for split in ("train", "validation"):
        ds = make_set(data_root, split)
        parts = [ds._filtered(i)[0].shape[0] for i in G.RECORD[split]]       # the augmentation keeps the count
        assert min(parts) < n_part < max(parts), (split, parts)
        distinct = [len(np.unique(GOLDEN[G.record_key(split, k, "pcd_full")], axis=0)) for k in range(len(G.RECORD[split]))]
        assert min(distinct) < G.NUM_POINTS == max(distinct), (split, distinct)


def test_batch_matches_collated_items(fake, data_root):
    h, batched = fake
    ds = make_set(data_root, "train")
    for indices in ([2], [4, 0], [1, 3, 0, 2]):
        np.random.seed(5)
        torch.manual_seed(5)
        items = [ds[i] for i in indices]
        np.random.seed(5)
        torch.manual_seed(5)
        b = ds.batch(indices)
        ref = D.SparseSegmentCollation()(items)
        assert b["filename"] == ref["filename"] == tuple(ds.points_datapath[i] for i in indices)
        for key in ("pcd_full", "mean", "std", "pcd_part"):
            assert b[key].dtype == torch.float32 and torch.equal(b[key], ref[key]), key
    assert batched == [4]                     # only the batch of at least FPS_CLUSTER_MIN_SCANS scans sampled in one launch


def test_random_draws_in_reference_order(fake, data_root):
    """augment() draws rotate (1 uniform), perturbation (3 normals), scale (1 uniform), flip (1 random) from numpy's global
    generator; the shuffle is one torch.randperm per sample from torch's global generator"""
    np.random.seed(3)
    D.augment(torch.zeros((4, 3), dtype=torch.float64))
    after = np.random.get_state()[1].copy(), np.random.get_state()[2]
    np.random.seed(3)
    np.random.uniform(), np.random.randn(3), np.random.uniform(0.95, 1.05, 1), np.random.random()
    assert (np.random.get_state()[1] == after[0]).all() and np.random.get_state()[2] == after[1]

    ds = make_set(data_root, "validation")
    torch.manual_seed(9)
    ds[0]
    after = torch.get_rng_state()
    torch.manual_seed(9)
    part, full = ds._filtered(0)
    keep, _ = fake_samples_backend.restate_viewpoint(part.numpy(), full.numpy(), D.VIEWPOINT_VOXEL)
    torch.randperm(int(keep.sum()))
    assert torch.equal(torch.get_rng_state(), after)


def test_augment_rounding():
    """rotation and perturbation are stored as float32, the scale acts on fp64 and the flip negates y"""
    np.random.seed(1)
    p = torch.tensor([[1.1, -2.3, 0.7], [30.25, 4.5, -1.0]], dtype=torch.float64)
    got = D.augment(p.clone()).numpy()
    np.random.seed(1)
    a = np.random.uniform() * 2 * np.pi
    R1 = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    q = (p.numpy() @ R1).astype(np.float32).astype(np.float64)
    ang = np.clip(0.06 * np.random.randn(3), -0.18, 0.18)
    Rx = np.array([[1, 0, 0], [0, np.cos(ang[0]), -np.sin(ang[0])], [0, np.sin(ang[0]), np.cos(ang[0])]])
    Ry = np.array([[np.cos(ang[1]), 0, np.sin(ang[1])], [0, 1, 0], [-np.sin(ang[1]), 0, np.cos(ang[1])]])
    Rz = np.array([[np.cos(ang[2]), -np.sin(ang[2]), 0], [np.sin(ang[2]), np.cos(ang[2]), 0], [0, 0, 1]])
    q = (q @ (Rz @ (Ry @ Rx))).astype(np.float32).astype(np.float64)
    q = q * np.random.uniform(0.95, 1.05, 1)[0]
    if np.random.random() > 0.5:
        q[:, 1] = -q[:, 1]
    assert (np.abs(got - q) <= 2 * np.spacing(np.abs(q).astype(np.float32))).all()


def test_repeat_is_elementwise():
    p = torch.tensor([[0.0, 0, 0], [1, 1, 1], [2, 2, 2]], dtype=torch.float64)
    got = D.repeat_rows(p, 2)
    assert torch.equal(got, torch.from_numpy(p.numpy().repeat(2, 0)))
    assert got[:, 0].tolist() == [0, 0, 1, 1, 2, 2]


def test_test_split_reads_no_map(fake, data_root, tmp_path):
    root = str(tmp_path / "nomap")
    shutil.copytree(data_root, root)
    os.remove(os.path.join(root, "dataset", "sequences", "08", "map_clean.npy"))
    ds = make_set(root, "test")
    assert ds.cache_maps == {"08": None}
    np.random.seed(G.SEED)
    torch.manual_seed(G.SEED)
    for k, i in enumerate(G.RECORD["test"]):
        assert_close_to_golden("test", k, ds[i])
    with pytest.raises(FileNotFoundError):
        make_set(root, "validation")


def test_empty_partial_scan_raises(fake, data_root, tmp_path):
    root = str(tmp_path / "empty")
    shutil.copytree(data_root, root)
    lab = os.path.join(root, "dataset", "sequences", "08", "labels", "000001.label")
    np.full(os.path.getsize(lab) // 4, 252, dtype=np.uint32).tofile(lab)          # every point a moving object
    ds = make_set(root, "validation")
    with pytest.raises(ValueError, match="08/velodyne/000001.bin"):
        ds[1]
    ds[0]


def test_empty_viewpoint_map_raises(fake, data_root, tmp_path):
    root = str(tmp_path / "far")
    shutil.copytree(data_root, root)
    m = os.path.join(root, "dataset", "sequences", "08", "map_clean.npy")
    np.save(m, np.load(m) + np.float32(200.0))          # no map point within max_range of any pose
    ds = make_set(root, "validation")
    with pytest.raises(ValueError, match="08/velodyne/000000.bin"):
        ds[0]


def test_data_module_splits(fake, data_root):
    cfg = {"data": {"data_dir": data_root, "resolution": G.RESOLUTION, "split": "train", "train": ["00", "01"], "validation": ["08"],
                    "num_points": G.NUM_POINTS, "max_range": G.MAX_RANGE, "dataset_norm": False, "std_axis_norm": False},
           "train": {"batch_size": 2, "num_workers": 4}}
    dm = D.dataloaders["KITTI"](cfg, device="cpu")
    tr, va, te = dm.train_dataloader(), dm.val_dataloader(), dm.test_dataloader()
    assert (tr.dataset.split, tr.dataset.seqs, tr.batch_size, type(tr.sampler)) == ("train", ["00", "01"], 2, RandomSampler)
    assert (va.dataset.split, va.dataset.seqs, va.batch_size, type(va.sampler)) == ("validation", ["08"], 1, SequentialSampler)
    assert (te.dataset.split, te.dataset.seqs, te.batch_size, type(te.sampler)) == ("validation", ["08"], 2, SequentialSampler)
    assert tr.num_workers == va.num_workers == te.num_workers == 0
    batches = list(te)
    assert [len(b["filename"]) for b in batches] == [2, 1]
    assert batches[0]["pcd_full"].shape == (2, G.NUM_POINTS, 3) and batches[0]["pcd_part"].shape == (2, G.NUM_POINTS // 10, 3)
    assert batches[1]["filename"] == (te.dataset.points_datapath[2],)
