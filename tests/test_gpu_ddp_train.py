"""Data-parallel training on the GPU: 2-rank training steps of each network (two processes on one GPU over gloo), wrapped as the CLIs
wrap them, whose first-step gradients meet the relative-L2 1e-2 rule against one process over the union of the ranks' clouds with
plain batch norm (the gradient of (1/W) sum_r loss_r with batch statistics over the union), whose BN running statistics are the
union's, and which leave identical parameters on both ranks and on a rerun; and both training CLIs under torchrun, whose checkpoints resume in one process and load in
the test CLIs.  With two or more GPUs the CLI test also runs with one device per rank (NCCL)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

import fake_sync_bn_backend as fake
import sync_bn_ranks

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_refine_sample_goldens as GR  # noqa: E402
import make_sample_goldens as GD  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("which,n", [("refine", 4000), ("diffusion", 4000)])
def test_two_rank_steps_are_identical_across_ranks_and_runs(tmp_path, which, n):
    a = fake.run_ranks(sync_bn_ranks.train_rank, 2, tmp_path / "a", which, n, "cuda", 2, fake=False)
    b = fake.run_ranks(sync_bn_ranks.train_rank, 2, tmp_path / "b", which, n, "cuda", 2, fake=False)
    assert a[0]["params"].tobytes() == a[1]["params"].tobytes()
    assert a[0]["params"].tobytes() == b[0]["params"].tobytes()
    assert a[0]["sync_bns"] > 0 and a[0]["plain_bns"] == 0
    ref = sync_bn_ranks.union_first_step(which, n, 2, "cuda")
    rel = [(g - r).norm().item() / r.norm().item() for g, r in zip(a[0]["grads"], ref["grads"]) if r.norm() > 1e-12]
    assert len(rel) > 0.9 * len(ref["grads"])
    assert max(rel) <= 1e-2, sorted(rel)[-3:]
    for k, v in ref["running"].items():
        np.testing.assert_allclose(a[0]["running"][k].numpy(), v.numpy(), rtol=1e-4, atol=1e-6, err_msg=k)


def _torchrun(args, env_extra, timeout=900):
    env = {**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), **env_extra}
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "2", "-m", *args]
    p = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        # SIGTERM first: torchrun's agent then stops its workers, which run in sessions of their own and would outlive a SIGKILL of
        # the agent; SIGKILL only if the agent has not exited after that
        p.terminate()
        try:
            out, _ = p.communicate(timeout=120)
        except subprocess.TimeoutExpired:
            p.kill()
            out, _ = p.communicate()
        raise AssertionError(f"torchrun did not finish within {timeout} s:\n{out}")
    assert p.returncode == 0, out
    return out


def _one_process(module, args):
    from click.testing import CliRunner
    res = CliRunner().invoke(module.main, args, catch_exceptions=False)
    assert res.exit_code == 0, res.output
    return res.output


def _diffusion_cfg(root):
    return {"experiment": {"id": "ddp_diff"},
            "data": {"data_dir": root, "resolution": 0.05, "dataloader": "KITTI", "split": "train", "train": GD.TRAIN,
                     "validation": GD.VALIDATION, "num_points": GD.NUM_POINTS, "max_range": 50.0, "dataset_norm": False,
                     "std_axis_norm": False},
            "train": {"uncond_prob": 0.1, "uncond_w": 6.0, "batch_size": 1, "num_workers": 4, "lr": 1e-4, "max_epoch": 20},
            "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 50, "reg_weight": 5.0},
            "model": {"out_dim": 96}}


def _refine_cfg(root):
    return {"experiment": {"id": "ddp_refine"},
            "data": {"data_dir": root, "resolution": 0.05, "split": "train", "train": GR.TRAIN, "validation": GR.VALIDATION,
                     "scan_window": GR.SCAN_WINDOW, "num_points": GR.NUM_POINTS},
            "train": {"batch_size": 1, "num_workers": 4, "mode": "refine", "up_factor": 6, "lr": 1e-3, "max_epoch": 3}}


def _cli_case(tmp_path, which, env):
    from lidiff_b200.tools import test_completion, test_refine, train_diffusion, train_refine
    if which == "diffusion":
        cfg, module, key = _diffusion_cfg(GD.make_dataset(str(tmp_path / "kitti"))), train_diffusion, "train/loss_mse"
    else:
        cfg, module, key = _refine_cfg(GR.make_dataset(str(tmp_path / "kitti"))), train_refine, "train/cd_loss"
    path = tmp_path / "config.yaml"
    path.write_text(yaml.safe_dump(cfg))
    out = tmp_path / "ckpt"
    log = _torchrun([module.__name__, "-c", str(path), "--out", str(out), "--max-steps", "2"], env)
    steps = [line for line in log.splitlines() if key in line]
    assert len(steps) == 2, log                                          # rank 0 prints, once per step
    saved = [line.split()[-1] for line in log.splitlines() if line.startswith("saved ")]
    assert saved, log
    ck = torch.load(saved[-1], weights_only=False)
    assert ck["global_step"] == 2 and ck["hyper_parameters"]["train"]["n_gpus"] == 2
    assert not any(k.startswith("module.") for k in ck["state_dict"])
    # a second run writes the same weights
    log2 = _torchrun([module.__name__, "-c", str(path), "--out", str(tmp_path / "ckpt2"), "--max-steps", "2"], env)
    ck2 = torch.load([line.split()[-1] for line in log2.splitlines() if line.startswith("saved ")][-1], weights_only=False)
    for k, v in ck["state_dict"].items():
        assert torch.equal(v, ck2["state_dict"][k]), k
    # resume in one process, then the test CLI
    res = _one_process(module, ["-c", str(path), "--out", str(out), "-ckpt", saved[-1], "--max-steps", "1"])
    assert [line for line in res.splitlines() if key in line][0].startswith(f"epoch {ck['epoch'] + 1} step 2 ")
    resumed = [line.split()[-1] for line in res.splitlines() if line.startswith("saved ")][-1]
    if which == "diffusion":
        res = _one_process(test_completion, ["-w", resumed, "-c", str(path), "--out", str(tmp_path / "gen"), "-T", "2"])
        assert "CD Mean:" in res
    else:
        res = _one_process(test_refine, ["-w", resumed, "-c", str(path), "--loader", "val"])
        assert "val/cd_loss mean over" in res


@pytest.mark.parametrize("which", ["diffusion", "refine"])
def test_cli_under_torchrun_two_ranks_on_one_gpu(tmp_path, which):
    _cli_case(tmp_path, which, {"CUDA_VISIBLE_DEVICES": os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]})


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs (one device per rank)")
@pytest.mark.parametrize("which", ["diffusion", "refine"])
def test_cli_under_torchrun_nccl_one_gpu_per_rank(tmp_path, which):
    _cli_case(tmp_path, which, {})
