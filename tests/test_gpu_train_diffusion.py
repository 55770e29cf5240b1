"""Diffusion training on the GPU: lb2_segment_dot against the restatement of its order (bit for bit), against fp64 (an explicit
fp32 bound) and on rerun; the gate's gradients on the golden scan's maps; grad-mode against no-grad MinkUNetDiff; whole-network
gradients against the CPU path; repeatable steps; learning; and the train_diffusion CLI end to end."""
import copy
import math
import os
import sys

import numpy as np
import pytest
import torch
import yaml
from click.testing import CliRunner

from lidiff_b200 import _lib
from lidiff_b200 import me as ME
from lidiff_b200.gate import GateMul

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_sample_goldens as G  # noqa: E402
import segment_dot_reference as sdr  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
R = sdr.R


def segment_dot(a, b, order, offsets):
    out = torch.full((len(offsets) - 1, a.shape[1]), 7.0, device=DEV)
    dev = lambda v: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).to(DEV)   # noqa: E731
    _lib.get_handle(DEV).segment_dot(dev(a), dev(b), dev(order), dev(np.asarray(offsets, np.int64)), out)
    return out.cpu().numpy()


def lengths_of(shape, g):
    if shape == "one_segment":
        return [1_000_000]
    if shape == "one_row_each":
        return [1] * 20_000
    if shape == "empties":
        return [0, 0, 5, 0, 0, 0, 2 * R + 3, 1, 0, R, 0, 0]
    if shape == "chunk_edges":
        return [R - 1, R, R + 1, R - 1, 1, R, R + 1, 2 * R, 2 * R - 1, 2 * R + 1]
    if shape == "power_law":
        return list(np.minimum((g.pareto(0.7, 3000) * 3).astype(np.int64), 150_000))
    raise KeyError(shape)


def check(a, b, order, offsets):
    got = segment_dot(a, b, order, offsets)
    want = sdr.emulate(a, b, order, offsets)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()
    assert np.array_equal(got.view(np.uint32), segment_dot(a, b, order, offsets).view(np.uint32))
    ref, bound = sdr.exact_and_bound(a, b, order, offsets)
    assert (np.abs(got - ref) <= bound).all(), (np.abs(got - ref) / np.maximum(bound, 1e-300)).max()


@pytest.mark.parametrize("shape", ["one_segment", "one_row_each", "empties", "chunk_edges", "power_law"])
def test_segment_dot_over_segment_shapes(shape):
    g = np.random.default_rng(len(shape))
    offsets = np.concatenate([[0], np.cumsum(lengths_of(shape, g))]).astype(np.int64)
    n, c = int(offsets[-1]), 32
    a = g.standard_normal((n, c)).astype(np.float32)
    b = g.standard_normal((n, c)).astype(np.float32)
    check(a, b, g.permutation(n), offsets)


@pytest.mark.parametrize("c", [1, 3, 32, 96, 256])
@pytest.mark.parametrize("use_b", [True, False], ids=["dot", "sum"])
def test_segment_dot_over_channel_counts(c, use_b):
    g = np.random.default_rng(c)
    offsets = np.concatenate([[0], np.cumsum([3, 0, 5 * R + 7, R, 1, 40, 0, 2 * R + 1])]).astype(np.int64)
    n = int(offsets[-1])
    a = (g.standard_normal((n, c)) * np.exp(g.uniform(-6, 6, (n, 1)))).astype(np.float32)
    b = g.standard_normal((n, c)).astype(np.float32) if use_b else None
    check(a, b, g.permutation(n), offsets)
    check(a, b, None, offsets)                                  # order NULL: the rows as they lie


def test_segment_dot_empty_inputs_and_rejected_widths():
    h = _lib.get_handle(DEV)
    off = torch.zeros(4, dtype=torch.int64, device=DEV)
    out = torch.full((3, 8), 7.0, device=DEV)
    h.segment_dot(torch.empty(0, 8, device=DEV), None, torch.empty(0, dtype=torch.int64, device=DEV), off, out)       # no rows
    assert (out == 0).all()
    out = torch.full((0, 8), 7.0, device=DEV)
    h.segment_dot(torch.ones(4, 8, device=DEV), None, None, torch.zeros(1, dtype=torch.int64, device=DEV), out)      # nseg == 0
    for c in (0, 257):
        with pytest.raises(RuntimeError, match=r"lb2_segment_dot failed \(-1\)"):
            h.segment_dot(torch.ones(4, c, device=DEV), None, None, torch.tensor([0, 4], device=DEV), torch.empty(1, max(c, 1), device=DEV))
    with pytest.raises(RuntimeError, match="fp32"):
        h.segment_dot(torch.ones(4, 8, device=DEV, dtype=torch.float64), None, None, torch.tensor([0, 4], device=DEV), torch.empty(1, 8, device=DEV))


def test_a_non_finite_row_reaches_its_own_segment_only():
    g = np.random.default_rng(5)
    lengths = [R + 9, 3 * R, 17, 2 * R]
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    n = int(offsets[-1])
    a = g.standard_normal((n, 8)).astype(np.float32)
    b = g.standard_normal((n, 8)).astype(np.float32)
    order = g.permutation(n)
    clean = segment_dot(a, b, order, offsets)
    a[order[offsets[1] + R + 2], 3] = np.nan                  # segment 1, a piece in the middle
    a[order[offsets[2] + 1], 5] = np.inf                      # segment 2
    got = segment_dot(a, b, order, offsets)
    assert np.isnan(got[1, 3]) and np.isinf(got[2, 5])
    mask = np.ones(got.shape, bool)
    mask[1, 3] = mask[2, 5] = False
    assert np.array_equal(got[mask].view(np.uint32), clean[mask].view(np.uint32))


# ---- the gate on the golden scan's maps -----------------------------------------------------------------------------------------
def golden_points():
    z = np.load(os.path.join(HERE, "golden", "step_000123.npz"))
    return torch.from_numpy(z["part"]).float()[None]


@pytest.mark.parametrize("uncond", [False, True], ids=["cond", "uncond"])
@pytest.mark.parametrize("ts,c", [(1, 32), (4, 128), (16, 256)])
def test_gate_gradients_on_the_golden_scan(uncond, ts, c):
    from lidiff_b200.minkunet import MinkUNetDiff
    from lidiff_b200.tools.train_diffusion import points_to_tensor
    pts = golden_points()
    g = torch.Generator().manual_seed(ts)
    full = torch.cat([pts, pts + 0.3 * torch.randn(pts.shape, generator=g)])           # two scans
    part = torch.zeros(2, 1800, 3) if uncond else full[:, ::10]
    xs = points_to_tensor(full, 0.05, DEV).sparse()
    cm = xs.coordinate_manager
    x_lvl = ME.SparseTensor(torch.empty(cm.level(ts).n, 1, device=DEV), coordinate_manager=cm, tensor_stride=ts)
    pf = points_to_tensor(part, 0.05, DEV).sparse()
    p_lvl = ME.SparseTensor(torch.empty(pf.coordinate_manager.level(16).n, 1, device=DEV), coordinate_manager=pf.coordinate_manager,
                            tensor_stride=16)
    idx = MinkUNetDiff._match_index(None, x_lvl, p_lvl)
    m, mp = x_lvl.F.shape[0], p_lvl.F.shape[0]
    assert (mp == 2) == uncond
    assert torch.equal(x_lvl.C[:, 0].long(), p_lvl.C[:, 0].long()[idx])                 # every row matched within its scan
    gd = torch.Generator(device=DEV).manual_seed(c)
    X = torch.randn(m, c, device=DEV, generator=gd).requires_grad_(True)
    T = torch.randn(mp, c, device=DEV, generator=gd).requires_grad_(True)
    Gr = torch.randn(m, c, device=DEV, generator=gd) * 1e-3
    y = GateMul.apply(X, T, idx)
    (y * Gr).sum().backward()
    X64, T64 = X.detach().double().requires_grad_(True), T.detach().double().requires_grad_(True)
    y64 = X64 * T64[idx]
    (y64 * Gr.double()).sum().backward()
    assert torch.equal(y.detach(), (X * T[idx]).detach())
    assert (X.grad.double() - X64.grad).abs().max().item() <= 2.0 ** -23 * X64.grad.abs().max().item()
    S1 = torch.zeros(mp, c, dtype=torch.float64, device=DEV).index_add_(0, idx, (Gr.double() * X.detach().double()).abs())
    longest = int(torch.bincount(idx).max())
    n_ops = 1 + min(longest, R) + longest // R + 2
    assert ((T.grad.double() - T64.grad).abs() <= ((1 + 2.0 ** -24) ** n_ops - 1) * S1 + 1e-40).all()


# ---- the whole network ---------------------------------------------------------------------------------------------------------
def _cfg(root=None, **train):
    return {"experiment": {"id": "diff_test"},
            "data": {"data_dir": root, "resolution": 0.05, "dataloader": "KITTI", "split": "train", "train": G.TRAIN,
                     "validation": G.VALIDATION, "num_points": G.NUM_POINTS, "max_range": 50.0, "dataset_norm": False, "std_axis_norm": False},
            "train": {"uncond_prob": 0.1, "uncond_w": 6.0, "batch_size": 2, "num_workers": 4, "lr": 1e-4, "max_epoch": 20, **train},
            "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 50, "reg_weight": 5.0},
            "model": {"out_dim": 96}}


def _batch(seed=0, n=3000, part=0):
    g = torch.Generator().manual_seed(seed)
    full = torch.randn(2, n, 3, generator=g) * torch.tensor([3.0, 3.0, 0.5])
    return {"pcd_full": full, "pcd_part": full[:, : max(n // 10, part)].clone()}


def _grads(nets, batch, cfg, device, seed=3):
    from lidiff_b200.tools import train_diffusion as T
    nets = nets.to(device).train()
    nets.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    noise = torch.randn(batch["pcd_full"].shape)           # the same noise on either device: drawn on the host and injected
    real = torch.randn
    torch.randn = lambda *a, **k: noise.to(k.get("device", "cpu"))
    try:
        out = T.training_forward(nets, batch, cfg, T.sqrt_one_minus_alphas_cumprod(cfg), torch.device(device))
    finally:
        torch.randn = real
    out["loss"].backward()
    return out["loss"].item(), {k: p.grad.detach().double().cpu().clone() for k, p in nets.named_parameters()}


@pytest.mark.parametrize("uncond", [False, True], ids=["cond", "uncond"])
def test_network_gradients_match_the_cpu_path_and_repeat_bit_for_bit(monkeypatch, uncond):
    from lidiff_b200.tools import train_diffusion as T
    cfg = _cfg(uncond_prob=2.0 if uncond else -1.0)
    torch.manual_seed(0)
    nets = T.DiffusionNets(cfg)
    nets_cpu = copy.deepcopy(nets)
    batch = _batch(n=8000, part=2500)
    l1, g1 = _grads(nets, batch, cfg, DEV)
    l2, g2 = _grads(nets, batch, cfg, DEV)
    assert l1 == l2
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    import fake_diffusion_backend
    fake_diffusion_backend.install(monkeypatch)                # the same networks on the CPU path
    l3, g3 = _grads(nets_cpu, batch, cfg, "cpu")
    assert abs(l1 - l3) <= 1e-4 * abs(l3)
    rel = {k: (g1[k] - g3[k]).norm().item() / max(g3[k].norm().item(), 1e-30) for k in g1 if g3[k].norm() > 1e-12}
    worst = max(rel.values())
    print("worst relative L2", sorted(((v, k) for k, v in rel.items()), reverse=True)[:3])
    # stated tolerance: relative L2 of every parameter's gradient <= 1e-2 (measured on an H100: 5.9e-3 conditional, 2.0e-3
    # unconditional).  The part cloud is large enough for the encoder's batch statistics: with 300 part points per scan they are
    # taken over a few dozen coarse rows and amplify the FP16x3 difference between the two forwards to 2.2e-2
    assert worst <= 1e-2, worst


def test_grad_mode_forward_agrees_with_no_grad_under_the_1e3_rule():
    from lidiff_b200.tools import train_diffusion as T
    cfg = _cfg()
    torch.manual_seed(1)
    nets = T.DiffusionNets(cfg).to(DEV).eval()                 # eval: the no-grad forward must not move the running statistics
    batch = _batch(1)
    x_full = T.points_to_tensor(batch["pcd_full"], 0.05, DEV)
    x_part = T.points_to_tensor(batch["pcd_part"], 0.05, DEV)
    t = torch.tensor([100, 700], device=DEV)
    with torch.no_grad():
        a = nets(x_full, x_part, t)
    b = nets(x_full, x_part, t)
    assert b.requires_grad and not a.requires_grad
    ratio = ((b.detach() - a).abs() / (a.abs() + a.pow(2).mean().sqrt())).max().item()
    print("grad-mode vs no-grad max |a - b| / (|b| + rms)", ratio)
    assert ratio <= 1e-3, ratio


def test_a_training_step_repeats_bit_for_bit():
    from lidiff_b200.tools import train_diffusion as T
    cfg = _cfg()
    somac = T.sqrt_one_minus_alphas_cumprod(cfg)
    states = []
    for _ in range(2):
        torch.manual_seed(0)
        torch.cuda.manual_seed(0)
        nets = T.DiffusionNets(cfg).to(DEV).train()
        opt, _ = T.make_optimizer(nets, cfg)
        for _ in range(2):
            T.train_step(nets, opt, _batch(2), cfg, somac, torch.device(DEV))
        states.append({k: v.clone() for k, v in nets.state_dict().items()})
    for k in states[0]:
        assert torch.equal(states[0][k], states[1][k]), k


def test_adam_steps_lower_the_loss_of_one_batch():
    from lidiff_b200.tools import train_diffusion as T
    cfg = _cfg()
    somac = T.sqrt_one_minus_alphas_cumprod(cfg)
    torch.manual_seed(0)
    nets = T.DiffusionNets(cfg).to(DEV).train()
    opt, _ = T.make_optimizer(nets, cfg)
    batch = _batch(3, n=6000)
    logs = []
    for _ in range(50):
        torch.manual_seed(1)                                    # a fixed batch: the same noise and time steps at every step
        torch.cuda.manual_seed(1)
        logs.append({k: v.item() for k, v in T.train_step(nets, opt, batch, cfg, somac, torch.device(DEV)).items() if k != "uncond"})
    print("first step", logs[0], "last step", logs[-1])
    assert all(math.isfinite(v) for log in logs for v in log.values())
    # the objective falls (measured on an H100: DESIGN.md §3); loss_mse alone need not in the first steps, while the
    # regulariser pulls the output's standard deviation from its initial value towards 1
    assert logs[-1]["loss"] <= 0.8 * logs[0]["loss"], (logs[0], logs[-1])


# ---- the CLI -------------------------------------------------------------------------------------------------------------------
def test_train_cli_resume_and_completion_cli(tmp_path):
    from lidiff_b200.tools import test_completion, train_diffusion
    root = G.make_dataset(str(tmp_path / "kitti"))
    path = tmp_path / "config.yaml"
    path.write_text(yaml.safe_dump(_cfg(root)))
    out = tmp_path / "ckpt"
    res = CliRunner().invoke(train_diffusion.main, ["-c", str(path), "--out", str(out), "--max-steps", "3"], catch_exceptions=False)
    assert res.exit_code == 0, res.output
    steps = [line for line in res.output.splitlines() if "train/loss_mse" in line]
    assert len(steps) == 3 and all(math.isfinite(float(line.split()[-1])) for line in steps)
    saved = [line.split()[-1] for line in res.output.splitlines() if line.startswith("saved ")]
    c = torch.load(saved[-1], weights_only=False)
    assert c["global_step"] == 3 and len(c["optimizer_states"]) == 1 and len(c["lr_schedulers"]) == 1
    res = CliRunner().invoke(train_diffusion.main, ["-c", str(path), "--out", str(out), "-ckpt", saved[-1], "--max-steps", "1"],
                             catch_exceptions=False)
    assert res.exit_code == 0, res.output
    steps = [line for line in res.output.splitlines() if "train/loss_mse" in line]
    assert len(steps) == 1 and steps[0].startswith(f"epoch {c['epoch'] + 1} step 3 ")
    resumed = [line.split()[-1] for line in res.output.splitlines() if line.startswith("saved ")][-1]
    assert torch.load(resumed, weights_only=False)["global_step"] == 4
    res = CliRunner().invoke(test_completion.main, ["-w", resumed, "-c", str(path), "--out", str(tmp_path / "gen"), "-T", "2"],
                             catch_exceptions=False)
    assert res.exit_code == 0, res.output
    assert "Saving " in res.output and "CD Mean:" in res.output
