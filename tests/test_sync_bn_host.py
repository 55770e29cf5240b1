"""The synchronised batch norm on the CPU: the restatement of lb2_sync_bn_* (tests/sync_bn_reference.py) pinned by hand-checked
cases and against fp64, gloo runs of 2 and 3 ranks on the CPU fake that give the bits of one process over the concatenated rows, and
convert_sync_batchnorm."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import fake_sync_bn_backend as fake
import sync_bn_ranks
import sync_bn_reference as R
from lidiff_b200 import me as ME


# ---- the restatement, by hand ------------------------------------------------------------------------------------------------
def test_words_of_a_hand_checked_channel():
    x = np.array([[1.0], [2.0], [3.0], [4.0]], dtype=np.float32)
    mw = R.fwd_max(x)
    assert mw.tolist() == [np.float32(4.0).view(np.uint32), 0]
    sw = R.fwd_sum(x, mw)                              # 4 < 2^3: s = 59, S = 10 * 2^59 = (10 * 2^27) * 2^32 + 0
    assert sw.tolist() == [10 << 27, 0, 4]
    mean, qw = R.fwd_sumsq(x, mw, sw)
    assert mean.tolist() == [2.5]
    # B = 4 + 2.5 < 2^3: t = 59; d = -1.5, -0.5, 0.5, 1.5; sum d^2 = 5 -> 5 * 2^118 = limb 3 holds 5 * 2^22
    assert qw.tolist() == [0, 0, 0, 5 << 22]
    var, invstd, y, rm, rv = R.fwd_apply(x, mw, sw, mean, qw, np.float32([2.0]), np.float32([0.5]), 1e-5, 0.1, np.float32([1.0]),
                                         np.float32([1.0]))
    assert var.tolist() == [1.25]
    assert invstd[0] == 1.0 / math.sqrt(1.25 + 1e-5)
    assert y[:, 0].tolist() == [np.float32(((v - 2.5) * invstd[0]) * 2.0 + 0.5) for v in (1.0, 2.0, 3.0, 4.0)]
    assert rm.tolist() == [np.float32(0.9 + 0.25)]
    assert rv.tolist() == [np.float32(0.9 * 1.0 + 0.1 * (1.25 * 4.0 / 3.0))]


def test_square_limbs_are_the_digits_of_the_exact_square():
    g = np.random.default_rng(0)
    p = np.concatenate([g.integers(-(1 << 62), 1 << 62, 2000), [0, 1, -1, 1 << 62, -(1 << 62), (1 << 32) - 1, 1 << 32]])
    # fwd_sumsq's limb arithmetic (p = a 2^32 + b) against Python's exact square
    for v in p:
        a = np.uint64(abs(int(v)))
        want = abs(int(v)) ** 2
        hi, lo = a >> np.uint64(32), a & np.uint64(R.M32)
        bb, ab, aa = lo * lo, hi * lo, hi * hi
        l0 = bb & np.uint64(R.M32)
        t1 = (bb >> np.uint64(32)) + ((ab << np.uint64(1)) & np.uint64(R.M32))
        t2 = (aa & np.uint64(R.M32)) + (ab >> np.uint64(31)) + (t1 >> np.uint64(32))
        l3 = (aa >> np.uint64(32)) + (t2 >> np.uint64(32))
        got = int(l0) + (int(t1 & np.uint64(R.M32)) << 32) + (int(t2 & np.uint64(R.M32)) << 64) + (int(l3) << 96)
        assert got == want


def test_constant_zero_subnormal_and_non_finite_channels():
    n = 50
    x = np.zeros((n, 5), np.float32)
    x[:, 0] = 3.7                                        # constant: mean exact, var 0, y = beta
    x[:, 1] = 0.0                                        # zeros
    x[:, 2] = np.float32(1e-44) * np.arange(n)           # subnormals
    x[:, 3] = np.linspace(-1, 1, n)
    x[7, 3] = np.nan
    x[:, 4] = np.linspace(-1, 1, n)
    x[9, 4] = -np.inf
    f = R.forward([x], np.ones(5, np.float32), np.full(5, 0.25, np.float32))
    assert f["mean"][0] == np.float64(np.float32(3.7)) and f["var"][0] == 0.0
    assert (f["ys"][0][:, 0] == np.float32(0.25)).all() and (f["ys"][0][:, 1] == np.float32(0.25)).all()
    sub = x[:, 2].astype(np.float64)
    assert f["mean"][2] == sub.mean() and abs(f["var"][2] - sub.var()) <= 1e-15 * sub.var()
    for j in (3, 4):
        assert np.isnan(f["mean"][j]) and np.isnan(f["var"][j]) and np.isnan(f["ys"][0][:, j]).all()
    assert np.isfinite(f["ys"][0][:, :3]).all()
    dy = np.ones((n, 5), np.float32)
    dy[3, 0] = np.inf
    b = R.backward([dy], [x], f, np.ones(5, np.float32))
    assert np.isnan(b["dxs"][0][:, 0]).all() and np.isnan(b["dxs"][0][:, 3:]).all() and np.isfinite(b["dxs"][0][:, 1:3]).all()
    assert np.isnan(b["dgammas"][0][0]) and np.isfinite(b["dgammas"][0][1:3]).all()


def _exact_stats(col):
    fr = [Fraction(float(v)) for v in col]
    m = sum(fr) / len(fr)
    return m, sum((v - m) ** 2 for v in fr) / len(fr)


@pytest.mark.parametrize("case", ["normal", "outlier", "offset"])
def test_statistics_within_the_stated_bound_of_exact_arithmetic(case):
    g = np.random.default_rng(1)
    n = 3000
    x = g.standard_normal((n, 3)).astype(np.float32)
    if case == "outlier":                                # max 1e4, sigma 1e-3
        x = (x * 1e-3).astype(np.float32)
        x[5] = 1e4
    elif case == "offset":                               # sigma 2^-20 max|x|
        x = (1000.0 + x * 1000.0 * 2.0 ** -20).astype(np.float32)
    f = R.forward([x], None, None)
    for j in range(3):
        m, v = _exact_stats(x[:, j])
        M = float(np.abs(x[:, j]).max())
        B = M + abs(f["mean"][j])
        assert abs(Fraction(f["mean"][j]) - m) <= Fraction(2.0 ** -62 * M) + Fraction(2.0 ** -53) * abs(m)
        bound = 2.0 ** -50 * float(v) + 2.0 ** -59 * B * math.sqrt(float(v)) + 2.0 ** -100 * B * B
        assert abs(Fraction(f["var"][j]) - v) <= Fraction(bound)


# ---- ranks on the CPU fake -----------------------------------------------------------------------------------------------------
def _problem(n, c, seed):
    g = np.random.default_rng(seed)
    x = (g.standard_normal((n, c)) * g.uniform(0.01, 10, c) + g.uniform(-5, 5, c)).astype(np.float32)
    x[: n // 50, 0] = 300.0                              # an outlier block
    dy = g.standard_normal((n, c)).astype(np.float32)
    gamma, beta = g.uniform(0.5, 2, c).astype(np.float32), g.uniform(-1, 1, c).astype(np.float32)
    return x, dy, gamma, beta


@pytest.mark.parametrize("world", [2, 3])
def test_ranks_give_the_bits_of_one_process_over_the_concatenation(tmp_path, world):
    n, c = 403, 32
    x, dy, gamma, beta = _problem(n, c, world)
    perm, idx = fake.split_rows(n, world, seed=10 + world)
    res = fake.run_ranks(sync_bn_ranks.bn_rank, world, tmp_path, [x[i] for i in idx], [dy[i] for i in idx], gamma, beta, "cpu")
    one = R.forward([x], gamma, beta, 1e-5, 0.1, np.zeros(c, np.float32), np.ones(c, np.float32))
    back = R.backward([dy], [x], one, gamma)
    y = sync_bn_ranks.rows_of([r["y"] for r in res], perm, n)
    dx = sync_bn_ranks.rows_of([r["dx"] for r in res], perm, n)
    assert y.tobytes() == one["ys"][0].tobytes()
    assert dx.tobytes() == back["dxs"][0].tobytes()
    for r in res:
        for k in ("mean", "var", "invstd"):
            assert r[k].tobytes() == one[k].tobytes()
        assert r["running_mean"].tobytes() == one["running_mean"].tobytes()
        assert r["running_var"].tobytes() == one["running_var"].tobytes()
        assert r["num_batches_tracked"] == 1
    # the local parameter gradients add up to the one-process sums (within their own fp32 roundings)
    np.testing.assert_allclose(sum(r["dgamma"].astype(np.float64) for r in res), back["dgammas"][0], rtol=1e-5, atol=1e-4)

    # against fp64 autograd of (1 / W) sum_r loss_r with batch statistics over the union
    x64 = torch.from_numpy(x).double().requires_grad_(True)
    g64 = torch.from_numpy(gamma).double().requires_grad_(True)
    b64 = torch.from_numpy(beta).double().requires_grad_(True)
    y64 = torch.nn.functional.batch_norm(x64, None, None, g64, b64, training=True, eps=1e-5)
    ((y64 * torch.from_numpy(dy).double()).sum() / world).backward()
    np.testing.assert_allclose(y, y64.detach().numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(dx, world * x64.grad.numpy(), rtol=1e-5, atol=1e-5)
    for r in res:
        np.testing.assert_allclose(r["avg_dgamma"], g64.grad.numpy(), rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(r["avg_dbeta"], b64.grad.numpy(), rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(r["running_var"], 0.9 + 0.1 * x.astype(np.float64).var(0, ddof=1), rtol=1e-6)


def test_convert_keeps_modules_keys_and_single_process_bits(monkeypatch):
    fake.install(monkeypatch)
    torch.manual_seed(0)
    net = torch.nn.Sequential(ME.MinkowskiBatchNorm(8), torch.nn.Sequential(ME.MinkowskiReLU(), ME.MinkowskiBatchNorm(4)))
    bns = [net[0].bn, net[1][1].bn]
    keys = list(net.state_dict().keys())
    params = [id(p) for p in net.parameters()]
    conv = ME.MinkowskiSyncBatchNorm.convert_sync_batchnorm(net)
    assert isinstance(conv[0], ME.MinkowskiSyncBatchNorm) and isinstance(conv[1][1], ME.MinkowskiSyncBatchNorm)
    assert conv[0].bn is bns[0] and conv[1][1].bn is bns[1]
    assert list(conv.state_dict().keys()) == keys and [id(p) for p in conv.parameters()] == params
    # no process group: exactly nn.BatchNorm1d, in training and in eval mode
    x = torch.randn(100, 8)
    ref = torch.nn.BatchNorm1d(8)
    ref.load_state_dict(bns[0].state_dict())
    for mode in (True, False):
        conv.train(mode)
        ref.train(mode)
        got = conv[0](ME.SparseTensor(x, coordinate_manager=object())).F
        assert got.detach().numpy().tobytes() == ref(x).detach().numpy().tobytes()
    sync = ME.MinkowskiSyncBatchNorm(4)
    assert ME.MinkowskiSyncBatchNorm.convert_sync_batchnorm(sync) is sync


# ---- data sharding and data-parallel training steps -------------------------------------------------------------------------
class _Items(torch.utils.data.Dataset):
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return i


@pytest.mark.parametrize("n,world,batch", [(10, 2, 2), (11, 3, 2), (7, 4, 3), (1, 2, 1)])
def test_shards_have_equal_batch_counts_and_cover_the_dataset(n, world, batch):
    from lidiff_b200 import ddp
    base = torch.utils.data.DataLoader(_Items(n), batch_size=batch, shuffle=True, collate_fn=list)
    assert ddp.sharded(base, ddp.Run(0, 1, torch.device("cpu")), shuffle=True) is base           # single process: untouched
    for epoch in (0, 1):
        seen, counts = [], []
        for rank in range(world):
            loader = ddp.sharded(base, ddp.Run(rank, world, torch.device("cpu")), shuffle=True)
            ddp.set_epoch(loader, epoch)
            batches = list(loader)
            counts.append(len(batches))
            seen += [i for b in batches for i in b]
        assert len(set(counts)) == 1
        assert set(seen) == set(range(n)) and len(seen) == world * math.ceil(n / world)
    # validation: no shuffle, rank r takes every world-th sample from r of the list padded by repeating its start
    val = ddp.sharded(base, ddp.Run(1, world, torch.device("cpu")), shuffle=False)
    assert [i for b in val for i in b] == (list(range(n)) * world)[: world * math.ceil(n / world)][1::world]


@pytest.mark.parametrize("which,n", [("refine", 40), ("diffusion", 60)])
def test_two_rank_training_steps_leave_identical_parameters(tmp_path, which, n):
    res = fake.run_ranks(sync_bn_ranks.train_rank, 2, tmp_path, which, n, "cpu", 2)
    assert res[0]["params"].tobytes() == res[1]["params"].tobytes()
    assert res[0]["state_keys"] == res[1]["state_keys"] and not any(k.startswith("module.") for k in res[0]["state_keys"])
    assert res[0]["sync_bns"] > 0 and res[0]["plain_bns"] == 0                # the wrapped model synchronises every BN
