"""Host logic of refinement training on the CPU fake (tests/fake_train_backend.py): for every layer kind the input gradient's
adjoint map and weight transform, and the weight gradient's map, reproduce fp64 autograd through oracle.me_cpu.conv; the voxel mean
and slice gradients match autograd through the oracle's; and the train_refine checkpoint resumes bit for bit."""
import numpy as np
import pytest
import torch

import fake_train_backend
from lidiff_b200 import me as ME
from lidiff_b200 import metrics
from oracle import me_cpu as ome


def cloud(n=400, seed=0):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(n, 3, generator=g) * torch.tensor([0.6, 0.6, 0.2])
    coords = torch.cat([torch.zeros(n, 1), torch.round(pts / 0.1)], 1)
    return pts, coords


# (layer class, cin, cout, kernel_size, stride, input tensor stride)
LAYERS = [
    ("conv", 32, 32, 3, 1, 1),          # 3x3x3 stride 1: the mirrored offsets
    ("conv", 32, 64, 2, 2, 1),          # k2 s2: the transposed map
    ("transpose", 64, 32, 2, 2, 2),     # k2 s2 transposed: the strided map
    ("conv", 32, 64, 1, 1, 1),          # 1x1: the identity with W^T
    ("conv", 384, 256, 3, 1, 2),        # a 384-channel cat input: two launches of 256 + 128 output channels
    ("conv", 192, 128, 1, 1, 2),        # 192 = 128 + 64
]


@pytest.mark.parametrize("kind,cin,cout,ks,stride,ts", LAYERS)
def test_conv_gradients_match_fp64_autograd(monkeypatch, kind, cin, cout, ks, stride, ts):
    fake_train_backend.install(monkeypatch)
    pts, coords = cloud()
    cls = ME.MinkowskiConvolutionTranspose if kind == "transpose" else ME.MinkowskiConvolution
    torch.manual_seed(1)
    layer = cls(cin, cout, kernel_size=ks, stride=stride, dimension=3)
    field = ME.TensorField(pts, coords)
    cm = field.sparse().coordinate_manager
    og = ome.TensorField(pts, coords).sparse().geom
    m = cm.level(ts).n
    assert m == og.stride_level(ts).shape[0]
    g = torch.Generator().manual_seed(2)
    X = torch.randn(m, cin, generator=g).requires_grad_(True)
    y = layer(ME.SparseTensor(X, coordinate_manager=cm, tensor_stride=ts))
    G = torch.randn(y.F.shape, generator=g)
    (y.F * G).sum().backward()

    X64 = X.detach().double().requires_grad_(True)
    W64 = layer.kernel.detach().double().requires_grad_(True)
    y64 = ome.conv(ome.SparseTensor(X64, og, ts), W64, ks, stride, kind == "transpose").F
    np.testing.assert_allclose(y.F.detach().double().numpy(), y64.detach().numpy(), rtol=1e-5, atol=1e-5)
    (y64 * G.double()).sum().backward()
    for got, ref in ((X.grad, X64.grad), (layer.kernel.grad, W64.grad)):
        assert got.shape == ref.shape
        scale = ref.abs().max().item()
        np.testing.assert_allclose(got.double().numpy(), ref.numpy(), rtol=0, atol=1e-5 * scale)
    # inner-product identity <conv(x), g> = <x, dgrad(g)>
    lhs = (y64.detach() * G.double()).sum().item()
    rhs = (X64.detach() * X.grad.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + 1.0)


def test_input_gradient_is_skipped_for_inputs_without_grad(monkeypatch):
    h = fake_train_backend.install(monkeypatch)
    pts, coords = cloud()
    layer = ME.MinkowskiConvolution(32, 32, kernel_size=3, stride=1, dimension=3)
    x = ME.TensorField(torch.randn(pts.shape[0], 32), coords).sparse()
    calls = []
    monkeypatch.setattr(type(layer), "_input_grad", lambda *a: calls.append(a))
    layer(x).F.sum().backward()
    assert calls == [] and layer.kernel.grad is not None


def test_voxel_mean_and_slice_gradients(monkeypatch):
    fake_train_backend.install(monkeypatch)
    pts, coords = cloud(600, 3)
    F = torch.randn(pts.shape[0], 5, dtype=torch.float32).requires_grad_(True)
    field = ME.TensorField(F, coords)
    s = field.sparse()
    sl = s.slice(field).F
    g = torch.randn(sl.shape)
    (sl * g).sum().backward()
    F64 = F.detach().double().requires_grad_(True)
    of = ome.TensorField(F64, coords)
    os_ = of.sparse()
    (os_.slice(of) * g.double()).sum().backward()
    np.testing.assert_allclose(F.grad.double().numpy(), F64.grad.numpy(), rtol=1e-6, atol=1e-6)


def test_chamfer_gradient_matches_autograd_of_the_closed_form(monkeypatch):
    fake_train_backend.install(monkeypatch)
    g = np.random.default_rng(0)
    x = torch.from_numpy(g.uniform(-1, 1, (2, 60, 3))).requires_grad_(True)
    y = torch.from_numpy(g.uniform(-1, 1, (2, 40, 3)))
    loss, _ = metrics.chamfer_distance(x, y)
    loss.backward()
    d = ((x.detach()[:, :, None] - y[:, None]) ** 2).sum(-1)
    ix, iy = d.argmin(2), d.argmin(1)
    x64 = x.detach().clone().requires_grad_(True)
    ref = sum(((x64[b] - y[b][ix[b]]) ** 2).sum(-1).mean() + ((y[b] - x64[b][iy[b]]) ** 2).sum(-1).mean() for b in range(2)) / 2
    ref.backward()
    np.testing.assert_allclose(x.grad.numpy(), x64.grad.numpy(), rtol=1e-12, atol=1e-15)


def _cfg():
    return {"experiment": {"id": "T"}, "data": {"resolution": 0.05}, "train": {"lr": 1e-3, "up_factor": 2, "max_epoch": 1}}


def _batch(seed):
    g = torch.Generator().manual_seed(seed)
    full = torch.randn(1, 300, 3, generator=g, dtype=torch.float64) * 2
    return {"pcd_noise": (full[:, :150] + 0.05 * torch.randn(1, 150, 3, generator=g, dtype=torch.float64)).float(),
            "pcd_full": full.float()}


def test_checkpoint_resume_reproduces_the_next_step(monkeypatch, tmp_path):
    fake_train_backend.install(monkeypatch)
    from lidiff_b200.minkunet import MinkUNet
    from lidiff_b200.tools import train_refine as T
    from lidiff_b200.tools.test_refine import load_refine_net
    cfg, dev = _cfg(), torch.device("cpu")
    torch.manual_seed(0)
    net = MinkUNet(in_channels=3, out_channels=6)
    opt = T.make_optimizer(net, cfg)
    T.train_step(net, opt, _batch(1), cfg, dev)
    path = T.checkpoint_path(str(tmp_path), cfg, 0)
    T.save_checkpoint(path, net, opt, cfg, 0, 1)
    T.train_step(net, opt, _batch(2), cfg, dev)

    torch.manual_seed(5)
    net2 = MinkUNet(in_channels=3, out_channels=6)
    opt2 = T.make_optimizer(net2, cfg)
    ck = T.load_checkpoint(path, net2, opt2)
    assert ck["epoch"] == 0 and ck["global_step"] == 1 and ck["hyper_parameters"] == cfg
    assert path.endswith("T_epoch=00.ckpt")
    T.train_step(net2, opt2, _batch(2), cfg, dev)
    for (k, a), (_, b) in zip(net.state_dict().items(), net2.state_dict().items()):
        assert torch.equal(a, b), k
    loaded = load_refine_net(path, 2, dev)
    assert all(k.startswith("model_refine.") for k in torch.load(path, weights_only=False)["state_dict"])
    assert set(loaded.state_dict()) == set(net.state_dict())
