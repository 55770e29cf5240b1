"""Records what the reference (PRBonn/LiDiff) computes on the import shims, so the tests that compare against it run without its
source tree:

    python tests/golden/make_reference_goldens.py REF       # REF = a checkout of the reference  -> tests/golden/reference_on_shims.npz
                                                              #                                       tests/golden/reference_names.json

  * reference_on_shims.npz: `DiffCompletion(diff, refine, T=2, s=6).complete_scan(raw)` of the reference's inference script, run
    unchanged on the shims with the CPU stand-in backend (tests/fake_backend.py), two consecutive scans under torch seed 123 (the
    checkpoints and the scan are seeded, see tests/test_reference_on_shims.py);
  * reference_names.json: the parameter names and shapes of the reference's MinkGlobalEnc / MinkUNetDiff / MinkUNet, the names its
    inference script imports from the shimmed packages, and what its metrics module (lidiff/utils/metrics.py) reports on a seeded
    pair of clouds.
"""
import importlib
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

SHIMMED = ("open3d", "natsort", "pytorch_lightning", "MinkowskiEngine", "diffusers", "pykeops")


def drop_lidiff():
    for k in [k for k in sys.modules if k == "lidiff" or k.startswith("lidiff.")]:
        sys.modules.pop(k)


def metrics_case():
    """the seeded clouds of test_shims.test_reference_metrics_module_runs_on_the_open3d_shim"""
    g = np.random.default_rng(3)
    gt = g.normal(size=(6000, 3)) * [12, 12, 1.0]
    pred = gt[g.choice(6000, 4000, replace=False)] + g.normal(size=(4000, 3)) * 0.05
    return gt, pred


def main(ref):
    import lidiff_b200.shims as sh
    sh.install()
    names = {}
    # ---- parameter names / shapes of the reference networks --------------------------------------------------------------
    spec = importlib.util.spec_from_file_location("ref_minkunet", os.path.join(ref, "lidiff/models/minkunet.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    names["state_dicts"] = {n: {k: list(v.shape) for k, v in getattr(mk, n)(in_channels=3, **kw).state_dict().items()}
                            for n, kw in (("MinkGlobalEnc", {}), ("MinkUNetDiff", {}), ("MinkUNet", {"out_channels": 18}))}
    # ---- the metrics module on the open3d shim ------------------------------------------------------------------------------
    import open3d as o3d
    sys.path.insert(0, ref)
    drop_lidiff()
    metrics = importlib.import_module("lidiff.utils.metrics")
    metrics.torch = torch                                     # the module uses `torch.Tensor` without importing torch
    gt, pred = metrics_case()
    pg, pp = o3d.geometry.PointCloud(gt), o3d.geometry.PointCloud(pred)
    cd, rm = metrics.ChamferDistance(), metrics.RMSE()
    cd.update(pg, pp); rm.update(pg, pp)
    pr = metrics.PrecisionRecall(0.05, 1.0, 20)
    pr.update(pg, pp)
    iou = metrics.CompletionIoU(voxel_sizes=[2.0, 1.0, 0.5])
    iou.update(pg, pp)
    names["metrics"] = {"chamfer": float(cd.compute()[0]), "rmse": float(rm.compute()[0]),
                        "precision_recall_f1_at_0.1": [float(v) for v in pr.compute_at_threshold(0.1)[:3]],
                        "auc": [float(v) for v in pr.compute_auc()], "iou": {str(k): float(v) for k, v in iou.compute().items()}}
    # ---- the inference script: what it binds from the shimmed packages --------------------------------------------------------
    drop_lidiff()
    mp = pytest.MonkeyPatch()
    import fake_backend
    from test_reference_on_shims import lightning_checkpoints, patch_for_cpu
    for m in SHIMMED:
        for k in [k for k in sys.modules if k == m or k.startswith(m + ".")]:
            sys.modules.pop(k)
    fake_backend.install(mp)
    mod = importlib.import_module("lidiff.tools.diff_completion_pipeline")
    imported = {}
    for gname, v in sorted(vars(mod).items()):
        src = getattr(v, "__name__", None) if isinstance(v, type(sys)) else getattr(v, "__module__", None)
        if src and (src.split(".")[0] in SHIMMED or src.startswith("lidiff_b200.shims")):
            imported[gname] = [src, None if isinstance(v, type(sys)) else v.__qualname__]
    names["pipeline_imports"] = imported
    names["pipeline_base"] = [b.__module__ + "." + b.__qualname__ for b in mod.DiffCompletion.__mro__[1:2]]
    # ---- complete_scan of the reference class, two scans ----------------------------------------------------------------------
    import tempfile
    from lidiff_b200.synth import synthetic_scan
    with tempfile.TemporaryDirectory() as tmp:
        patch_for_cpu(mp, mod, tmp)
        diff_path, refine_path = lightning_checkpoints(tmp, 2000)
        raw = synthetic_scan(9, beams=16, azimuths=256)
        r = mod.DiffCompletion(diff_path, refine_path, 2, 6.0)
        out = {"pre": r.preprocess_scan(raw).numpy()}
        torch.manual_seed(123)
        for scan_no in range(2):
            refined, post = r.complete_scan(raw)
            out[f"refined{scan_no}"], out[f"post{scan_no}"] = refined, post
    mp.undo()
    np.savez_compressed(os.path.join(HERE, "reference_on_shims.npz"), **out)
    json.dump(names, open(os.path.join(HERE, "reference_names.json"), "w"), indent=0)
    print({k: (v.dtype, v.shape) for k, v in out.items()})


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
