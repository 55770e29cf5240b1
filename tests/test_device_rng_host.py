"""Host logic of device_rng=True on the CPU fakes (tests/fake_rng_backend.py): the refinement and diffusion data modules give the
same batches as device_rng=False, and leave numpy's and torch's generators in the same states; numpy_randn / torch_randperm keep
their contracts at the edges (cached Gaussians, the all-host band, a too-short word stream, n = 0 and 1)."""
import os
import sys

import numpy as np
import pytest
import torch

import fake_rng_backend as FR
from lidiff_b200 import datasets as D
from lidiff_b200 import datasets_refine as DR
from lidiff_b200 import rng

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_refine_sample_goldens as GR  # noqa: E402
import make_sample_goldens as GD  # noqa: E402


@pytest.fixture(scope="module")
def refine_root(tmp_path_factory):
    return GR.make_dataset(str(tmp_path_factory.mktemp("kitti_refine")))


@pytest.fixture(scope="module")
def diffusion_root(tmp_path_factory):
    return GD.make_dataset(str(tmp_path_factory.mktemp("kitti_diffusion")))


def _run(loader_of, device_rng):
    np.random.seed(3)
    torch.manual_seed(3)
    batches = list(loader_of(device_rng))
    return batches, np.random.get_state(legacy=True), torch.get_rng_state()


def _assert_same(loader_of):
    host, np_h, t_h = _run(loader_of, False)
    dev, np_d, t_d = _run(loader_of, True)
    assert len(host) == len(dev) > 0
    for a, b in zip(host, dev):
        for k in a:
            assert (torch.equal(a[k], b[k]) if isinstance(a[k], torch.Tensor) else a[k] == b[k]), k
    assert np.array_equal(np_h[1], np_d[1]) and np_h[2:] == np_d[2:]
    assert torch.equal(t_h, t_d)


@pytest.mark.parametrize("which", ["train", "val", "test"])
def test_refine_loaders(refine_root, monkeypatch, which):
    FR.install_refine(monkeypatch)
    cfg = {"data": {"data_dir": refine_root, "resolution": GR.RESOLUTION, "split": "train", "train": GR.TRAIN,
                    "validation": GR.VALIDATION, "scan_window": GR.SCAN_WINDOW, "num_points": GR.NUM_POINTS},
           "train": {"batch_size": 2, "num_workers": 0, "mode": "refine"}}
    _assert_same(lambda dr: getattr(DR.TemporalKittiDataModule(cfg, device="cpu", device_rng=dr), f"{which}_dataloader")())


@pytest.mark.parametrize("which", ["train", "val", "test"])
def test_diffusion_loaders(diffusion_root, monkeypatch, which):
    FR.install_samples(monkeypatch)
    cfg = {"data": {"data_dir": diffusion_root, "resolution": GD.RESOLUTION, "split": "train", "train": GD.TRAIN,
                    "validation": GD.VALIDATION, "num_points": GD.NUM_POINTS, "max_range": GD.MAX_RANGE, "dataset_norm": False,
                    "std_axis_norm": False},
           "train": {"batch_size": 2, "num_workers": 0}}
    _assert_same(lambda dr: getattr(D.TemporalKittiDataModule(cfg, device="cpu", device_rng=dr), f"{which}_dataloader")())


@pytest.mark.parametrize("n,cached,band", [(0, True, 1 / 32), (1, True, 1 / 32), (1, False, 1 / 32), (2, True, 0.5), (7, False, 0.5),
                                           (2001, True, 1 / 32)])
def test_numpy_randn_contract(monkeypatch, n, cached, band):
    FR.install_refine(monkeypatch)
    a, b = np.random.RandomState(8), np.random.RandomState(8)
    for rs in (a, b):
        rs.randn(3 if cached else 2)
    got = rng.numpy_randn(n, device="cpu", random_state=a, band=band)
    assert np.array_equal(got.numpy().view(np.uint64), b.randn(n).view(np.uint64))
    sa, sb = a.get_state(legacy=True), b.get_state(legacy=True)
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def test_numpy_randn_draws_more_words_when_short(monkeypatch):
    """a stream cut below the needed attempts: the rest is drawn from the carried state and the result is unchanged"""
    FR.install_refine(monkeypatch)
    monkeypatch.setattr(rng, "_attempts", lambda pairs: pairs // 3)      # a third of the accepted attempts needed, at first
    a, b = np.random.RandomState(9), np.random.RandomState(9)
    got = rng.numpy_randn(3001, device="cpu", random_state=a)
    assert np.array_equal(got.numpy().view(np.uint64), b.randn(3001).view(np.uint64))
    sa, sb = a.get_state(legacy=True), b.get_state(legacy=True)
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


@pytest.mark.parametrize("n", [0, 1, 2, 700])
def test_torch_randperm_contract(monkeypatch, n):
    FR.install_refine(monkeypatch)
    g1, g2 = torch.Generator().manual_seed(n), torch.Generator().manual_seed(n)
    got = rng.torch_randperm(n, device="cpu", generator=g1)
    assert got.dtype == torch.int64 and torch.equal(got, torch.randperm(n, generator=g2))
    assert torch.equal(g1.get_state(), g2.get_state())


@pytest.mark.parametrize("key,arg,want", [(None, None, False), (False, None, False), (True, None, True), (True, False, False),
                                          (False, True, True), (None, True, True)])
def test_data_modules_take_the_switch_from_the_argument_or_the_config(refine_root, diffusion_root, monkeypatch, key, arg, want):
    """device_rng= wins; without it the config's data.device_rng decides, and a config without the key keeps the host draws"""
    FR.install_refine(monkeypatch)
    cfg_r = {"data": {"data_dir": refine_root, "resolution": GR.RESOLUTION, "split": "train", "train": GR.TRAIN,
                      "validation": GR.VALIDATION, "scan_window": GR.SCAN_WINDOW, "num_points": GR.NUM_POINTS},
             "train": {"batch_size": 2, "num_workers": 0, "mode": "refine"}}
    cfg_d = {"data": {"data_dir": diffusion_root, "resolution": GD.RESOLUTION, "split": "train", "train": GD.TRAIN,
                      "validation": GD.VALIDATION, "num_points": GD.NUM_POINTS, "max_range": GD.MAX_RANGE, "dataset_norm": False,
                      "std_axis_norm": False},
             "train": {"batch_size": 2, "num_workers": 0}}
    for cfg, module in ((cfg_r, DR), (cfg_d, D)):
        if key is not None:
            cfg["data"]["device_rng"] = key
        dm = module.TemporalKittiDataModule(cfg, device="cpu") if arg is None else \
            module.TemporalKittiDataModule(cfg, device="cpu", device_rng=arg)
        assert dm.device_rng is want
        for loader in (dm.train_dataloader(), dm.val_dataloader(), dm.test_dataloader()):
            assert loader.dataset.device_rng is want
