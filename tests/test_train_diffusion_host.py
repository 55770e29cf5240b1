"""Host logic of diffusion training on the CPU fake (tests/fake_diffusion_backend.py): the hoisted gate against the un-hoisted
expression in fp64, whole-network gradients of the training loss against fp64 autograd through the oracle, the restatement of
lb2_segment_dot's order against fp64, the order of the random draws and the unconditional switch, the learning-rate schedule and the
checkpoint."""
import numpy as np
import pytest
import torch

import fake_diffusion_backend
import segment_dot_reference as sdr
from lidiff_b200 import me as ME
from oracle import me_cpu as ome
from oracle import nets as onets


def _cloud(n, seed, batches=2, scale=(0.6, 0.6, 0.2)):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(batches, n, 3, generator=g) * torch.tensor(scale)
    return pts


def _cfg(**diff):
    return {"experiment": {"id": "D"}, "data": {"resolution": 0.05, "num_points": 300},
            "train": {"lr": 1e-3, "uncond_prob": 0.1, "uncond_w": 6.0, "max_epoch": 1, "batch_size": 2},
            "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 2, "reg_weight": 5.0, **diff},
            "model": {"out_dim": 96}}


def _batch(seed, batches=2, n=300):
    full = _cloud(n, seed, batches, (2.0, 2.0, 0.4))
    return {"pcd_full": full, "pcd_part": full[:, : n // 3].clone()}


# ---- the gate ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gate", [0, 4, 6], ids=["stage1", "up1", "up3"])
@pytest.mark.parametrize("uncond", [False, True], ids=["cond", "uncond"])
def test_hoisted_gate_matches_the_unhoisted_expression_in_fp64(monkeypatch, gate, uncond):
    fake_diffusion_backend.install(monkeypatch)
    from lidiff_b200.minkunet import MinkUNetDiff
    from lidiff_b200.tools.train_diffusion import points_to_tensor
    torch.manual_seed(gate)
    net = MinkUNetDiff(in_channels=3).double()
    name = net._GATES[gate]
    mlps = [getattr(net, f"latent_{name}"), getattr(net, f"{name}_temp"), getattr(net, f"latemp_{name}")]
    full, part = _cloud(400, 1), _cloud(60, 2)
    xs = points_to_tensor(full, 0.05, "cpu").sparse()
    ps = points_to_tensor(torch.zeros_like(part) if uncond else part, 0.05, "cpu").sparse()
    assert (ps.F.shape[0] == 2) == uncond                    # unconditional: one part voxel per scan
    g = torch.Generator().manual_seed(3)
    c = mlps[2][2].out_features
    X = torch.randn(xs.F.shape[0], c, generator=g, dtype=torch.float64)
    P = torch.randn(ps.F.shape[0], 256, generator=g, dtype=torch.float64)
    E = torch.randn(2, 96, generator=g, dtype=torch.float64)
    G = torch.randn(X.shape, generator=g, dtype=torch.float64)

    def run(hoisted):
        x, p, e = (v.clone().requires_grad_(True) for v in (X, P, E))
        net.zero_grad(set_to_none=True)
        xt, pt = xs._like(x), ps._like(p)
        if hoisted:
            y = net._gate(gate, xt, pt, e).F
        else:                                                # MinkUNetDiff._gate's expression, row by row over the voxels
            idx = net._match_index(xt, pt)
            t = mlps[1](e)[xs.C[:, 0].long()]
            q = mlps[0](p[idx])
            y = x * mlps[2](torch.cat((t, q) if name == "up1" else (q, t), -1))
        (y * G).sum().backward()
        return [y.detach(), x.grad, p.grad, e.grad] + [w.grad.clone() for m in mlps for w in m.parameters()]

    a, b = run(True), run(False)
    with torch.no_grad():
        np.testing.assert_allclose(net._gate(gate, xs._like(X), ps._like(P), E).F.numpy(), a[0].numpy(), rtol=1e-12, atol=1e-12)
    for u, v in zip(a, b):
        assert u.shape == v.shape
        np.testing.assert_allclose(u.numpy(), v.numpy(), rtol=1e-10, atol=1e-10 * max(v.abs().max().item(), 1.0))


def test_a_batch_without_part_rows_is_named(monkeypatch):
    fake_diffusion_backend.install(monkeypatch)
    from lidiff_b200.minkunet import MinkUNetDiff
    from lidiff_b200.tools.train_diffusion import points_to_tensor
    net = MinkUNetDiff(in_channels=3)
    xs = points_to_tensor(_cloud(100, 1), 0.05, "cpu").sparse()
    ps = points_to_tensor(_cloud(20, 2, batches=1), 0.05, "cpu").sparse()            # batch 1 has no part voxel
    x = xs._like(torch.randn(xs.F.shape[0], 32).requires_grad_(True))
    with pytest.raises(ValueError, match=r"no part voxel in batch \[1\]"):
        net._gate(0, x, ps._like(torch.randn(ps.F.shape[0], 256)), torch.randn(2, 96))


# ---- lb2_segment_dot's order ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_b", [True, False])
def test_segment_dot_restatement_against_fp64(use_b):
    g = np.random.default_rng(0)
    R = sdr.R
    lengths = [0, R - 1, R, R + 1, 0, 0, 1, 3 * R + 5, 1, 0]
    offsets = np.concatenate([[0], np.cumsum(lengths)])
    n = int(offsets[-1])
    a = g.standard_normal((n, 5)).astype(np.float32)
    b = g.standard_normal((n, 5)).astype(np.float32) if use_b else None
    order = g.permutation(n)
    got = sdr.emulate(a, b, order, offsets)
    ref, bound = sdr.exact_and_bound(a, b, order, offsets)
    assert (np.abs(got - ref) <= bound).all()
    assert (got[[0, 4, 5, 9]] == 0).all() and (bound[1] > 0).all()
    # the pieces: a segment that starts R - 1 rows into chunk 0 ... and one row in the middle of a chunk
    assert sdr.pieces_of(np.array([0, R - 1, 2 * R - 1])) == [[(0, R - 1)], [(R - 1, R), (R, 2 * R - 1)]]
    # a single piece is a sequential sum from +0
    v = np.array([[1.0], [2.0 ** -24], [2.0 ** -24]], np.float32)
    assert sdr.emulate(v, None, None, np.array([0, 3]))[0, 0] == np.float32(1.0)


# ---- whole-network gradients -----------------------------------------------------------------------------------------------------
class TrainNet(onets.Net):
    """the oracle's networks with batch normalisation in training mode (batch statistics, biased variance)"""

    def conv_bn(self, x, pconv, pbn, ks, stride=1, transposed=False, relu=True):
        y = ome.conv(x, self.sd[f"{pconv}.kernel"], ks, stride, transposed)
        F = (y.F - y.F.mean(0)) / torch.sqrt(y.F.var(0, unbiased=False) + 1e-5) * self.sd[f"{pbn}.bn.weight"] + self.sd[f"{pbn}.bn.bias"]
        return y.replace(torch.relu(F) if relu else F)


def _oracle_loss(nets, batch, cfg, noise, t, uncond):
    from lidiff_b200.tools.train_diffusion import sqrt_one_minus_alphas_cumprod
    sds = []
    for m in (nets.partial_enc, nets.model):
        sds.append({k: (v.detach().double().requires_grad_(True) if v.is_floating_point() else v) for k, v in m.state_dict().items()})
    enc, diff = TrainNet(sds[0], torch.float64), TrainNet(sds[1], torch.float64)

    def field(points):
        feats = ome.batched_coordinates(list(points), dtype=torch.float32)
        coords = feats.clone()
        coords[:, 1:] = torch.round(feats[:, 1:] / cfg["data"]["resolution"])
        return ome.TensorField(feats[:, 1:].double(), coords)

    x_full = field(batch["pcd_full"] + sqrt_one_minus_alphas_cumprod(cfg)[t][:, None, None] * noise)
    x_part = field(torch.zeros_like(batch["pcd_part"]) if uncond else batch["pcd_part"])
    out = diff.unet_diff(x_full, x_full.sparse(), enc.global_enc(x_part), t).reshape(t.shape[0], -1, 3)
    loss = ((out - noise.double()) ** 2).mean() + cfg["diff"]["reg_weight"] * (out.mean() ** 2 + (out.std() - 1.0) ** 2)
    loss.backward()
    grads = {f"{p}.{k}": v.grad for p, sd in zip(("partial_enc", "model"), sds) for k, v in sd.items()
             if v.is_floating_point() and v.grad is not None}
    return loss.item(), grads


@pytest.mark.parametrize("uncond", [False, True], ids=["cond", "uncond"])
def test_network_gradients_match_fp64_autograd_through_the_oracle(monkeypatch, uncond):
    fake_diffusion_backend.install(monkeypatch)
    from lidiff_b200.tools import train_diffusion as T
    cfg = _cfg()
    cfg["train"]["uncond_prob"] = 2.0 if uncond else -1.0
    torch.manual_seed(0)
    nets = T.DiffusionNets(cfg).train()
    batch = _batch(4)
    torch.manual_seed(7)
    out = T.training_forward(nets, batch, cfg, T.sqrt_one_minus_alphas_cumprod(cfg), torch.device("cpu"))
    assert out["uncond"] == uncond
    out["loss"].backward()
    torch.manual_seed(7)                                     # the draws of training_forward, in its order
    noise = torch.randn(batch["pcd_full"].shape)
    t = torch.randint(0, 1000, size=(2,))
    loss64, g64 = _oracle_loss(nets, batch, cfg, noise, t, uncond)
    assert abs(out["loss"].item() - loss64) <= 1e-4 * abs(loss64)
    got = {k: p.grad for k, p in nets.named_parameters()}
    assert set(got) == set(g64)
    worst = max((got[k].double() - g64[k]).norm().item() / max(g64[k].norm().item(), 1e-30) for k in got if g64[k].norm() > 1e-12)
    # fp32 batch normalisation, MLPs and loss against fp64 (the convolution products are fp64 on the fake): measured 1.1e-3 conditional, 2e-6 unconditional
    assert worst <= 5e-3, worst


# ---- the training step ---------------------------------------------------------------------------------------------------------
def test_random_draws_and_the_unconditional_switch(monkeypatch):
    from lidiff_b200.tools import train_diffusion as T
    calls, seen = [], {}
    real = {n: getattr(torch, n) for n in ("randn", "randint", "rand")}
    for n in real:
        monkeypatch.setattr(torch, n, lambda *a, _n=n, **k: (calls.append((_n, k.get("device"))), real[_n](*a, **k))[1])

    class Nets:
        def __call__(self, x_full, x_part, t):
            seen["part"] = x_part.F.clone()
            return torch.zeros(t.shape[0], x_full.F.shape[0] // t.shape[0], 3, requires_grad=True)

    monkeypatch.setattr(T, "points_to_tensor", lambda p, r, d: type("F", (), {"F": p.reshape(-1, 3)})())
    cfg, dev = _cfg(), torch.device("cpu")
    somac = T.sqrt_one_minus_alphas_cumprod(cfg)
    two, one = _batch(1), _batch(1, batches=1)
    for seed in range(40):
        torch.manual_seed(seed)
        calls.clear()
        out = T.training_forward(Nets(), two, cfg, somac, dev)
        assert calls == [("randn", dev), ("randint", None), ("rand", None)]
        torch.manual_seed(seed)
        real["randn"]((2, 300, 3)), real["randint"](0, 1000, size=(2,))
        want = not bool(real["rand"](1) > 0.1)
        assert out["uncond"] == want and bool((seen["part"] == 0).all()) == want
        seen[want] = True
        torch.manual_seed(seed)
        assert not T.training_forward(Nets(), one, cfg, somac, dev)["uncond"]      # never at B = 1
    assert seen.get(True) and seen.get(False)


def test_other_schedules_are_rejected_by_name():
    from lidiff_b200.tools import train_diffusion as T
    with pytest.raises(ValueError, match="'cosine'"):
        T.sqrt_one_minus_alphas_cumprod(_cfg(beta_func="cosine"))
    s = T.sqrt_one_minus_alphas_cumprod(_cfg())
    betas = np.linspace(3.5e-5, 0.007, 1000)
    np.testing.assert_allclose(s.numpy(), np.sqrt(1 - np.cumprod(1 - betas)), rtol=1e-3)      # fp32 1 - alphas_cumprod, as the reference


def test_learning_rate_halves_every_five_epochs():
    from lidiff_b200.tools import train_diffusion as T
    opt, sched = T.make_optimizer(torch.nn.Linear(2, 2), _cfg())
    lrs = []
    for epoch in range(11):
        lrs.append(opt.param_groups[0]["lr"])
        opt.step()
        T.end_epoch(sched, epoch)
    assert lrs == [1e-3] * 5 + [5e-4] * 5 + [2.5e-4]
    assert opt.defaults["betas"] == (0.9, 0.999)


def test_checkpoint_fields_resume_and_weights_only(monkeypatch, tmp_path):
    fake_diffusion_backend.install(monkeypatch)
    from lidiff_b200.tools import train_diffusion as T
    cfg, dev = _cfg(), torch.device("cpu")
    somac = T.sqrt_one_minus_alphas_cumprod(cfg)

    def fresh(seed):
        torch.manual_seed(seed)
        nets = T.DiffusionNets(cfg).train()
        return (nets, *T.make_optimizer(nets, cfg))

    def step(nets, opt, seed):
        torch.manual_seed(seed)
        T.train_step(nets, opt, _batch(seed), cfg, somac, dev)

    nets, opt, sched = fresh(0)
    step(nets, opt, 1)
    for epoch in range(5):
        T.end_epoch(sched, epoch)
    path = T.checkpoint_path(str(tmp_path), cfg, 4)
    assert path.endswith("D_epoch=04.ckpt")
    T.save_checkpoint(path, nets, opt, sched, cfg, 4, 1)
    step(nets, opt, 2)

    ck = torch.load(path, weights_only=False)
    assert set(ck) == {"state_dict", "optimizer_states", "lr_schedulers", "epoch", "global_step", "hyper_parameters"}
    assert {k.split(".")[0] for k in ck["state_dict"]} == {"partial_enc", "model"}
    assert ck["epoch"] == 4 and ck["global_step"] == 1 and ck["hyper_parameters"] == cfg

    nets2, opt2, sched2 = fresh(5)
    T.load_checkpoint(path, nets2, opt2, sched2)
    assert opt2.param_groups[0]["lr"] == 5e-4 and sched2.last_epoch == 1
    step(nets2, opt2, 2)
    for (k, a), (_, b) in zip(nets.state_dict().items(), nets2.state_dict().items()):
        assert torch.equal(a, b), k

    nets3, opt3, _ = fresh(6)
    T.load_checkpoint(path, nets3)                            # -w: the weights alone
    assert not opt3.state_dict()["state"] and opt3.param_groups[0]["lr"] == 1e-3
    for k, v in nets3.state_dict().items():
        assert torch.equal(v, ck["state_dict"][k]), k
    # the completion pipeline reads the file unchanged
    from lidiff_b200.pipeline import DiffCompletion
    pipe = DiffCompletion(path, None, 2, device="cpu", engine=False)
    assert torch.equal(pipe.model.last[0].weight, ck["state_dict"]["model.last.0.weight"])
