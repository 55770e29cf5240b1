"""device_rng=True samples equal device_rng=False samples row for row, with numpy's and torch's generators in the same states
afterwards, for the refinement and diffusion loaders on the recorded golden datasets, and still meet the goldens."""
import os
import sys

import numpy as np
import pytest
import torch

from lidiff_b200 import datasets as D
from lidiff_b200 import datasets_refine as R

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_refine_sample_goldens as GR  # noqa: E402
import make_sample_goldens as GD  # noqa: E402
import test_refine_samples_host as HR  # noqa: E402
import test_samples_host as HD  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def refine_root(tmp_path_factory):
    return GR.make_dataset(str(tmp_path_factory.mktemp("kitti_refine")))


@pytest.fixture(scope="module")
def diffusion_root(tmp_path_factory):
    return GD.make_dataset(str(tmp_path_factory.mktemp("kitti_diffusion")))


def _refine_cfg(root):
    return {"data": {"data_dir": root, "resolution": GR.RESOLUTION, "split": "train", "train": GR.TRAIN, "validation": GR.VALIDATION,
                     "scan_window": GR.SCAN_WINDOW, "num_points": GR.NUM_POINTS},
            "train": {"batch_size": 2, "num_workers": 0, "mode": "refine", "up_factor": 6}}


def _diffusion_cfg(root):
    return {"data": {"data_dir": root, "resolution": GD.RESOLUTION, "split": "train", "train": GD.TRAIN, "validation": GD.VALIDATION,
                     "num_points": GD.NUM_POINTS, "max_range": GD.MAX_RANGE, "dataset_norm": False, "std_axis_norm": False},
            "train": {"batch_size": 2, "num_workers": 0}}


def _run(loader_of, device_rng, seed=3):
    np.random.seed(seed)
    torch.manual_seed(seed)
    batches = list(loader_of(device_rng))
    return batches, np.random.get_state(legacy=True), torch.get_rng_state()


def _assert_same(loader_of):
    host, np_h, t_h = _run(loader_of, False)
    dev, np_d, t_d = _run(loader_of, True)
    assert len(host) == len(dev) > 0
    for a, b in zip(host, dev):
        assert a.keys() == b.keys()
        for k in a:
            if isinstance(a[k], torch.Tensor):
                assert torch.equal(a[k].cpu(), b[k].cpu()), k
            else:
                assert a[k] == b[k], k
    assert np_h[0] == np_d[0] and np.array_equal(np_h[1], np_d[1]) and np_h[2:] == np_d[2:]
    assert torch.equal(t_h, t_d)


@pytest.mark.parametrize("which", ["train", "val", "test"])
def test_refine_loaders_device_rng_equals_host(refine_root, which):
    cfg = _refine_cfg(refine_root)
    _assert_same(lambda dr: getattr(R.TemporalKittiDataModule(cfg, device=DEV, device_rng=dr), f"{which}_dataloader")())


@pytest.mark.parametrize("which", ["train", "val", "test"])
def test_diffusion_loaders_device_rng_equals_host(diffusion_root, which):
    cfg = _diffusion_cfg(diffusion_root)
    _assert_same(lambda dr: getattr(D.TemporalKittiDataModule(cfg, device=DEV, device_rng=dr), f"{which}_dataloader")())


@pytest.mark.parametrize("split", ["train", "validation", "test"])
def test_refine_device_rng_meets_the_goldens(refine_root, split):
    ds = R.TemporalKITTISet(refine_root, GR.SCAN_WINDOW, GR.split_seqs(split), GR.split_name(split), GR.RESOLUTION, GR.NUM_POINTS,
                            "refine", device=DEV, device_rng=True)
    np.random.seed(GR.SEED)
    torch.manual_seed(GR.SEED)
    for k, i in enumerate(GR.RECORD[split]):
        HR.assert_close_to_golden(split, k, ds[i])


@pytest.mark.parametrize("split", ["train", "validation", "test"])
def test_diffusion_device_rng_meets_the_goldens(diffusion_root, split):
    ds = D.TemporalKITTISet(diffusion_root, GD.split_seqs(split), split, GD.RESOLUTION, GD.NUM_POINTS, GD.MAX_RANGE, device=DEV,
                            device_rng=True)
    np.random.seed(GD.SEED)
    torch.manual_seed(GD.SEED)
    for k, i in enumerate(GD.RECORD[split]):
        HD.assert_close_to_golden(split, k, ds[i])


def _counting(monkeypatch):
    """count the device draws, so a run with the switch on is seen to use them"""
    from lidiff_b200 import rng
    calls = []
    for name in ("numpy_randn", "torch_randperm"):
        f = getattr(rng, name)
        monkeypatch.setattr(rng, name, lambda *a, _f=f, _n=name, **kw: calls.append(_n) or _f(*a, **kw))
    return calls


def _ply_bytes(root):
    out = {}
    for dp, _, fns in os.walk(root):
        for fn in sorted(fns):
            if fn.endswith(".ply"):
                with open(os.path.join(dp, fn), "rb") as f:
                    out[os.path.relpath(os.path.join(dp, fn), root)] = f.read()
    return out


@pytest.mark.parametrize("loader", ["val", "test"])
def test_refine_cli_takes_device_rng_from_the_config(refine_root, tmp_path, monkeypatch, loader):
    """test_refine with data.device_rng: true prints the same losses and writes the same PLYs as without it"""
    import yaml
    from click.testing import CliRunner
    from lidiff_b200.tools import test_refine as T
    calls = _counting(monkeypatch)
    runs = {}
    for dr in (False, True):
        cfg = _refine_cfg(refine_root)
        cfg["data"]["device_rng"] = dr
        path = tmp_path / f"config_{dr}.yaml"
        path.write_text(yaml.safe_dump(cfg))
        out = tmp_path / f"out_{dr}"
        res = CliRunner().invoke(T.main, ["--random-weights", "-c", str(path), "--loader", loader, "--out", str(out)],
                                 catch_exceptions=False)
        assert res.exit_code == 0, res.output
        runs[dr] = ([ln for ln in res.output.splitlines() if ln.startswith("batch ") or "cd_loss" in ln], _ply_bytes(out))
        assert (len(calls) > 0) == dr
    assert runs[False][0] and runs[False][0] == runs[True][0]
    assert runs[False][1] and runs[False][1] == runs[True][1]


def test_completion_cli_takes_device_rng_from_the_config(tmp_path, monkeypatch):
    """test_completion with data.device_rng: true writes the same completions and metrics as without it"""
    import yaml
    from click.testing import CliRunner
    from lidiff_b200.tools import test_completion as TC
    calls = _counting(monkeypatch)
    root = str(tmp_path / "data")
    os.makedirs(os.path.join(root, "dataset", "sequences"))
    GD.write_sequence(os.path.join(root, "dataset", "sequences", "08"), 2, 5)
    runs = {}
    for dr in (False, True):
        cfg = {"experiment": {"id": "t"}, "data": {"data_dir": root, "resolution": 0.05, "dataloader": "KITTI", "split": "train",
                                                   "train": ["00"], "validation": ["08"], "num_points": 20000, "max_range": 50.0,
                                                   "dataset_norm": False, "std_axis_norm": False, "device_rng": dr},
               "train": {"uncond_w": 6.0, "batch_size": 2, "num_workers": 4},
               "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 50}}
        path = tmp_path / f"config_{dr}.yaml"
        path.write_text(yaml.safe_dump(cfg))
        out = tmp_path / f"out_{dr}"
        res = CliRunner().invoke(TC.main, ["-c", str(path), "--out", str(out), "--random-weights", "-T", "3"], catch_exceptions=False)
        assert res.exit_code == 0, res.output
        runs[dr] = ([ln for ln in res.output.splitlines() if ":" in ln and any(k in ln for k in ("CD", "Precision", "Recall", "F-Score"))],
                    _ply_bytes(out))
        assert (len(calls) > 0) == dr
    assert runs[False][0] and runs[False][0] == runs[True][0]
    assert len(runs[False][1]) == 2 and runs[False][1] == runs[True][1]
