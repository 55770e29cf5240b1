"""The reference's OWN inference class on the import shims, against this repo's mirror `lidiff_b200.pipeline.DiffCompletion`:
the reference's `lidiff/tools/diff_completion_pipeline.py`, imported unchanged, constructed `DiffCompletion(diff_path, refine_path, T, s)`
from synthetic Lightning-format checkpoints (ctor: torch.load, save_hyperparameters, strict=False state-dict loads, scheduler
construction, exp_config.yaml) and ran `complete_scan(points)` end to end — preprocess (open3d FPS), points_to_tensor, the guided
sampling loop over the ME / diffusers shims, postprocess, refinement, 6x offsets — for two consecutive scans under torch seed 123
(the reference never resets its scheduler between scans).  tests/golden/make_reference_goldens.py recorded that run in
tests/golden/reference_on_shims.npz; the mirror must reproduce it bit for bit.

The CUDA library is replaced by tests/fake_backend.py (CPU stand-in under the same C-ABI-shaped handle) and `.cuda()` is a no-op:
what runs is every line of the mirror's host code and of the shims; the kernels themselves are covered by the -m gpu suites."""
import os

import numpy as np
import torch

import fake_backend
from conftest import make_scan

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_on_shims.npz")


def patch_for_cpu(monkeypatch, mod=None, cwd=None):
    """CPU stand-ins for what the reference's host code expects of a CUDA machine; mod: the imported inference script (its open3d
    farthest point sampling is a CUDA kernel in the shim, the oracle's CPU restatement stands in for it)"""
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.nn.Module, "cuda", lambda self, *a, **k: self)
    orig_to = torch.Tensor.to

    def to_cpu_instead_of_cuda(self, *a, **k):                                      # minkunet.py:395 `.to(torch.device('cuda'))`
        is_cuda = lambda x: (isinstance(x, torch.device) and x.type == "cuda") or (isinstance(x, str) and x.startswith("cuda"))
        a = tuple(torch.device("cpu") if is_cuda(x) else x for x in a)
        if is_cuda(k.get("device")):
            k["device"] = torch.device("cpu")
        return orig_to(self, *a, **k)
    monkeypatch.setattr(torch.Tensor, "to", to_cpu_instead_of_cuda)
    if cwd is not None:
        monkeypatch.chdir(cwd)                                                      # the ctor writes ./results/<exp>/exp_config.yaml
    if mod is not None:
        from oracle.pipeline import farthest_point_sample as fps_cpu

        def fps(self, n):
            pts = np.asarray(self.points)
            return type(self)(pts[fps_cpu(pts, int(n))])
        monkeypatch.setattr(mod.o3d.geometry.PointCloud, "farthest_point_down_sample", fps)


def lightning_checkpoints(tmp_path, n_points):
    """what LiDiff's training writes: {'hyper_parameters': config.yaml dict, 'state_dict': {<submodule>.<param>: tensor}}"""
    from oracle.pipeline import calibrated_state_dicts
    scan = make_scan(n_points // 10, 4)
    sds = calibrated_state_dicts(scan, seed=3)
    hp = {"experiment": {"id": "test"},
          "data": {"resolution": 0.05, "num_points": n_points, "max_range": 50.0, "dataloader": "KITTI"},
          "train": {"uncond_w": 6.0, "uncond_prob": 0.1, "lr": 1e-4},
          "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 50, "reg_weight": 5.0},
          "model": {"out_dim": 96}}
    sd_diff = {f"partial_enc.{k}": v for k, v in sds["enc"].items()}
    sd_diff.update({f"model.{k}": v for k, v in sds["diff"].items()})
    sd_ref = {f"model_refine.{k}": v for k, v in sds["refine"].items()}
    d, r = os.path.join(str(tmp_path), "diff_net.ckpt"), os.path.join(str(tmp_path), "refine_net.ckpt")
    torch.save({"epoch": 19, "hyper_parameters": hp, "state_dict": sd_diff}, d)
    torch.save({"epoch": 5, "hyper_parameters": hp, "state_dict": sd_ref}, r)
    return d, r


def test_reference_diffcompletion_runs_on_shims_and_equals_the_mirror(monkeypatch, tmp_path):
    from lidiff_b200.pipeline import DiffCompletion as Mirror
    from lidiff_b200.synth import range_filter, synthetic_scan
    fake_backend.install(monkeypatch)
    patch_for_cpu(monkeypatch, cwd=tmp_path)
    z = np.load(GOLD)
    n_points = 2000
    diff_path, refine_path = lightning_checkpoints(tmp_path, n_points)
    raw = synthetic_scan(9, beams=16, azimuths=256)                           # (4096, 3) incl. points the range filter drops
    mir = Mirror(diff_path, refine_path, 2, 6.0, device="cpu", engine=False)
    assert mir.hparams["data"]["num_points"] == n_points
    pre = torch.from_numpy(z["pre"])                                          # the reference's preprocess_scan(raw)
    assert tuple(pre.shape) == (1, n_points, 3) and pre.dtype == torch.float64
    assert pre.shape[1] == range_filter(raw).shape[0] or pre.shape[1] == n_points
    torch.manual_seed(123)
    res = []
    for scan_no in range(2):                                                  # second scan: multistep state carried over (no reset)
        refined, post = mir.complete_scan(pre, preprocessed=True)
        assert refined.shape == (6 * post.shape[0], 3) and np.isfinite(refined).all() and post.shape[0] > 0
        pa, ra = z[f"post{scan_no}"], z[f"refined{scan_no}"]
        assert pa.shape == post.shape and np.array_equal(pa, post), "diffusion result: reference class on shims vs mirror"
        assert np.array_equal(ra, refined), "refined result: reference class on shims vs mirror"
        res.append(post)
    assert not np.array_equal(res[0], res[1])                                 # the two scans drew different noise
