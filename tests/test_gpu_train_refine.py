"""Refinement training on the GPU: lb2_spconv_wgrad against an fp64 gather-GEMM on the real maps of tests/golden/step_000123.npz's
scan (the FP16x3 element-wise bound, bit-identical reruns), the input gradients on the adjoint maps, whole-network gradients against
the CPU path, grad-mode forward bits, the Chamfer gradient, learning, and the train_refine CLI end to end."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import yaml
from click.testing import CliRunner

from lidiff_b200 import _lib, metrics
from lidiff_b200 import me as ME

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_refine_sample_goldens as G  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"

# every (kvol, cin, cout) of MinkUNet(in_channels=3, out_channels=18), with the tensor stride it runs at
SHAPES = [(27, 3, 32, 1), (27, 32, 32, 1), (27, 32, 64, 4), (27, 64, 64, 4), (27, 64, 128, 8), (27, 128, 128, 8), (27, 128, 256, 16),
          (27, 256, 256, 16), (27, 384, 256, 8), (27, 192, 128, 4), (27, 128, 96, 2), (27, 96, 96, 2), (27, 128, 96, 1), (27, 96, 96, 1),
          (8, 32, 32, 1), (8, 32, 32, 2), (8, 64, 64, 4), (8, 128, 128, 8),                       # strided: input stride
          (-8, 256, 256, 16), (-8, 256, 128, 8), (-8, 128, 96, 4), (-8, 96, 96, 2),               # transposed: input stride
          (1, 32, 64, 2), (1, 64, 128, 4), (1, 128, 256, 8), (1, 384, 256, 8), (1, 192, 128, 4), (1, 128, 96, 2), (1, 128, 96, 1)]


def golden_field():
    z = np.load(os.path.join(HERE, "golden", "step_000123.npz"))
    pts = torch.from_numpy(z["part"]).float().to(DEV)
    coords = torch.cat([torch.zeros(pts.shape[0], 1, device=DEV), torch.round(pts / 0.05)], 1)
    field = ME.TensorField(pts, coords)
    field.sparse()
    return field.coordinate_manager


def layer_map(cm, kvol, ts):
    """(nbr or None, rows in, rows out)"""
    if kvol == 1:
        n = cm.level(ts).n
        return None, n, n
    if kvol == 27:
        return cm.kernel_map(ts, 3, 1, False), cm.level(ts).n, cm.level(ts).n
    if kvol == 8:
        return cm.kernel_map(ts, 2, 2, False), cm.level(ts).n, cm.level(2 * ts).n
    return cm.kernel_map(ts, 2, 2, True), cm.level(ts).n, cm.level(ts // 2).n


def gather_gemm64(X, Gr, nbr, kvol):
    X, Gr = X.double(), Gr.double()
    out = torch.zeros(kvol, X.shape[1], Gr.shape[1], dtype=torch.float64, device=DEV)
    for k in range(kvol):
        src = torch.arange(Gr.shape[0], device=DEV) if nbr is None else nbr[k].long()
        o = torch.nonzero(src >= 0)[:, 0]
        out[k] = X[src[o]].T @ Gr[o]
    return out


def wgrad(X, Gr, nbr, kvol):
    dw = torch.empty(kvol, X.shape[1], Gr.shape[1], device=DEV)
    _lib.get_handle(DEV).spconv_wgrad(X, Gr, nbr, kvol, dw)
    return dw


@pytest.mark.parametrize("kvol,cin,cout,ts", SHAPES, ids=lambda v: str(v))
def test_wgrad_within_the_fp16x3_bound_and_deterministic(kvol, cin, cout, ts):
    cm = golden_field()
    nbr, m_in, m_out = layer_map(cm, kvol, ts)
    kv = abs(kvol)
    g = torch.Generator(device=DEV).manual_seed(kv * 1000 + cin + cout)
    X = torch.randn(m_in, cin, device=DEV, generator=g).clamp(-1.99, 1.99)
    Gr = torch.randn(m_out, cout, device=DEV, generator=g) * 1e-4           # gradients are small: the pre-scale must hold them
    dw = wgrad(X, Gr, nbr, kv)
    assert torch.equal(dw.view(torch.int32), wgrad(X, Gr, nbr, kv).view(torch.int32))
    ref = gather_gemm64(X, Gr, nbr, kv)
    S1 = gather_gemm64(X.abs(), Gr.abs(), nbr, kv)
    k = min(14 - math.frexp(Gr.abs().max().item())[1], 126)
    sx = gather_gemm64(X.abs(), torch.ones(m_out, 1, device=DEV), nbr, kv)
    sg = gather_gemm64(torch.ones(m_in, 1, device=DEV), Gr.abs(), nbr, kv)
    floor = 1.001 * 2.0 ** -25 * (sg + 2.0 ** -k * sx)
    n_adds = math.ceil(m_out / 320) + 16                    # group folds of a chunk + the chunk reduction
    tau = 3.002 * 2.0 ** -22 + 60 * 2.0 ** -23 + n_adds * 2.0 ** -24
    err = (dw.double() - ref).abs()
    assert (err <= tau * S1 + floor).all(), (err / (tau * S1 + floor)).max().item()


def test_wgrad_rejects_unsupported_shapes():
    h = _lib.get_handle(DEV)
    x, g = torch.zeros(64, 40, device=DEV), torch.zeros(64, 48, device=DEV)
    with pytest.raises(RuntimeError, match="no kernel"):
        h.spconv_wgrad(x, g, None, 1, torch.empty(1, 40, 48, device=DEV))


# ---- input gradients through the ME surface ------------------------------------------------------------------------------
KINDS = [("conv", 64, 64, 3, 1, 1), ("conv", 32, 64, 2, 2, 1), ("transpose", 256, 128, 2, 2, 8), ("conv", 128, 256, 1, 1, 4),
         ("conv", 384, 256, 3, 1, 8), ("conv", 192, 128, 3, 1, 4)]


@pytest.mark.parametrize("kind,cin,cout,ks,stride,ts", KINDS, ids=lambda v: str(v))
def test_input_gradient_and_inner_product_identity(kind, cin, cout, ks, stride, ts):
    cm = golden_field()
    cls = ME.MinkowskiConvolutionTranspose if kind == "transpose" else ME.MinkowskiConvolution
    torch.manual_seed(cin + cout)
    layer = cls(cin, cout, kernel_size=ks, stride=stride, dimension=3).to(DEV)
    m = cm.level(ts).n
    X = torch.randn(m, cin, device=DEV).requires_grad_(True)
    y = layer(ME.SparseTensor(X, coordinate_manager=cm, tensor_stride=ts))
    Gr = torch.randn(y.F.shape, device=DEV) * 1e-3
    (y.F * Gr).sum().backward()
    # fp64 reference: the same convolution as a gather-GEMM per offset, differentiated by torch
    X64 = X.detach().double().requires_grad_(True)
    W = layer.kernel.detach().double()
    if W.dim() == 2:
        y64 = X64 @ W
    else:
        nbr = cm.kernel_map(ts, ks, stride, kind == "transpose")
        y64 = torch.zeros(y.F.shape, dtype=torch.float64, device=DEV)
        for k in range(W.shape[0]):
            o = torch.nonzero(nbr[k] >= 0)[:, 0]
            y64 = y64.index_add(0, o, X64[nbr[k][o].long()] @ W[k])
    (y64 * Gr.double()).sum().backward()
    scale = X64.grad.abs().max().item()
    assert (X.grad.double() - X64.grad).abs().max().item() <= 1e-5 * scale
    lhs = (y64.detach() * Gr.double()).sum().item()
    rhs = (X.detach().double() * X.grad.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (X.detach().double().abs() * X.grad.double().abs()).sum().item()


# ---- the whole network ---------------------------------------------------------------------------------------------------
def _net_and_batch(seed=0):
    from lidiff_b200.minkunet import MinkUNet
    torch.manual_seed(seed)
    net = MinkUNet(in_channels=3, out_channels=18)
    g = torch.Generator().manual_seed(seed)
    full = torch.randn(1, 3000, 3, generator=g) * torch.tensor([3.0, 3.0, 0.5])
    noise = full[:, :1000] + 0.05 * torch.randn(1, 1000, 3, generator=g)
    return net, {"pcd_noise": noise, "pcd_full": full}


def _grads(net, batch, device):
    from lidiff_b200.tools.train_refine import refine_forward
    net = net.to(device).train()
    net.zero_grad(set_to_none=True)
    _, loss = refine_forward(net, batch, 0.05, 6, torch.device(device))
    loss.backward()
    return loss.item(), {k: p.grad.detach().double().cpu().clone() for k, p in net.named_parameters()}


def test_network_gradients_match_the_cpu_path_and_repeat_bit_for_bit(monkeypatch):
    import copy
    net, batch = _net_and_batch()
    net_cpu = copy.deepcopy(net)
    l1, g1 = _grads(net, batch, DEV)
    l2, g2 = _grads(net, batch, DEV)
    assert l1 == l2
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    sys.path.insert(0, HERE)
    import fake_train_backend
    fake_train_backend.install(monkeypatch)           # the same network on the CPU path: fp64 convolution products
    l3, g3 = _grads(net_cpu, batch, "cpu")
    assert abs(l1 - l3) <= 1e-4 * abs(l3)
    worst = max((g1[k] - g3[k]).norm().item() / max(g3[k].norm().item(), 1e-30) for k in g1)
    # stated tolerance: relative L2 error of every parameter's gradient <= 1e-2 (measured 5.2e-3 on an H100).  The two forwards differ
    # at the FP16x3 level, enough to move a refined point across a near-tie of its Chamfer neighbour, which changes that point's
    # gradient outright rather than by a rounding error
    assert worst <= 1e-2, worst


def test_grad_mode_forward_is_bit_identical():
    net, batch = _net_and_batch(1)
    net = net.to(DEV).train()
    from lidiff_b200.tools.train_refine import refine_forward
    with torch.no_grad():
        a, la = refine_forward(net, batch, 0.05, 6, torch.device(DEV))
    b, lb = refine_forward(net, batch, 0.05, 6, torch.device(DEV))
    assert b.requires_grad and torch.equal(a, b.detach()) and torch.equal(la, lb.detach())


def test_chamfer_gradient_closed_form_with_ties():
    g = np.random.default_rng(4)
    y = np.round(g.uniform(-2, 2, (2, 500, 3)), 1).astype(np.float32)      # a 0.1 lattice: many exact ties
    x = np.concatenate([np.round(g.uniform(-2, 2, (2, 300, 3)) * 20) / 20, y[:, :60]], 1).astype(np.float32)
    xt = torch.from_numpy(x).to(DEV).requires_grad_(True)
    yt = torch.from_numpy(y).to(DEV).requires_grad_(True)
    loss, _ = metrics.chamfer_distance(xt, yt)
    loss.backward()
    gx, gy = np.zeros(x.shape), np.zeros(y.shape)
    for b in range(2):
        x64, y64 = x[b].astype(np.float64), y[b].astype(np.float64)
        d = ((x64[:, None] - y64[None]) ** 2).sum(-1)
        ix, iy = d.argmin(1), d.argmin(0)                                     # lowest index on ties
        nx, ny = x.shape[1], y.shape[1]
        r = x64 - y64[ix]
        gx[b] += 2 * r / nx / 2
        np.subtract.at(gy[b], ix, 2 * r / nx / 2)
        s = y64 - x64[iy]
        gy[b] += 2 * s / ny / 2
        np.subtract.at(gx[b], iy, 2 * s / ny / 2)
    np.testing.assert_allclose(xt.grad.double().cpu().numpy(), gx, rtol=0, atol=1e-7)
    np.testing.assert_allclose(yt.grad.double().cpu().numpy(), gy, rtol=0, atol=1e-7)


# ---- learning and the CLI ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def data_root(tmp_path_factory):
    return G.make_dataset(str(tmp_path_factory.mktemp("kitti")))


def _cfg(root, epochs=1):
    return {"experiment": {"id": "refine_test"},
            "data": {"data_dir": root, "resolution": 0.05, "split": "train", "train": G.TRAIN, "validation": G.VALIDATION,
                     "scan_window": G.SCAN_WINDOW, "num_points": G.NUM_POINTS},
            "train": {"batch_size": 2, "num_workers": 4, "mode": "refine", "up_factor": 6, "lr": 1e-3, "max_epoch": epochs}}


def test_adam_steps_lower_the_loss_of_one_window(data_root):
    from lidiff_b200.datasets_refine import TemporalKittiDataModule
    from lidiff_b200.minkunet import MinkUNet
    from lidiff_b200.tools import train_refine as T
    cfg = _cfg(data_root)
    np.random.seed(0)
    torch.manual_seed(0)
    batch = next(iter(TemporalKittiDataModule(cfg, device=DEV).train_dataloader()))
    net = MinkUNet(in_channels=3, out_channels=18).to(DEV).train()
    opt = T.make_optimizer(net, cfg)
    losses = [T.train_step(net, opt, batch, cfg, torch.device(DEV)).item() for _ in range(50)]
    print("losses", losses[0], losses[-1])
    assert all(math.isfinite(v) for v in losses)
    # stated factor: 50 steps lower the loss by at least 15 % (measured on an H100: 5.59 -> 4.22, 25 %)
    assert losses[-1] <= 0.85 * losses[0], (losses[0], losses[-1])


def test_train_cli_then_test_cli(data_root, tmp_path):
    from lidiff_b200.tools import test_refine, train_refine
    path = tmp_path / "config_refine.yaml"
    path.write_text(yaml.safe_dump(_cfg(data_root)))
    out = tmp_path / "ckpt"
    res = CliRunner().invoke(train_refine.main, ["-c", str(path), "--out", str(out)], catch_exceptions=False)
    assert res.exit_code == 0, res.output
    steps = [line for line in res.output.splitlines() if "train/cd_loss" in line]
    assert steps and all(math.isfinite(float(line.split()[-1])) for line in steps)
    ckpt = out / "refine_test_epoch=00.ckpt"
    assert ckpt.exists()
    c = torch.load(ckpt, weights_only=False)
    assert c["epoch"] == 0 and c["global_step"] == len(steps) and len(c["optimizer_states"]) == 1
    res = CliRunner().invoke(test_refine.main, ["-w", str(ckpt), "-c", str(path), "--loader", "val"], catch_exceptions=False)
    assert res.exit_code == 0, res.output
    assert "val/cd_loss mean over 1 batches" in res.output
    # resume: -ckpt continues at the next epoch; epoch 4 (the fifth) runs the validation pass
    cfg2 = _cfg(data_root, epochs=5)
    path.write_text(yaml.safe_dump(cfg2))
    res = CliRunner().invoke(train_refine.main, ["-c", str(path), "--out", str(out), "-ckpt", str(ckpt)], catch_exceptions=False)
    assert res.exit_code == 0, res.output
    assert next(line for line in res.output.splitlines() if "train/cd_loss" in line).startswith("epoch 1 ")
    assert "epoch 4 val/cd_loss" in res.output
    assert (out / "refine_test_epoch=04.ckpt").exists()
