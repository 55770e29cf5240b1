"""The synchronised batch norm's kernels on the GPU: every lb2_sync_bn_* output bit for bit against the restatement
(tests/sync_bn_reference.py) at every BN width of the three networks, from a few rows to 4 M, with constant, outlier, subnormal and
non-finite channels; identical bits on rerun and whatever the split of the rows into blocks; two gloo processes on one GPU that give
the bits of one process over the concatenated rows; and the compiler invariants of the kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import fake_sync_bn_backend as fake
import sync_bn_ranks
import sync_bn_reference as R
from lidiff_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def gpu_pass(xs, dys, gamma, beta, eps=1e-5, momentum=0.1, rm=None, rv=None):
    """the seven entry points over the row blocks `xs` (one "rank" each), the word arrays combined on the device between the calls;
    returns numpy copies of everything the calls wrote"""
    h = _lib.get_handle(DEV)
    xs, dys = [_t(x) for x in xs], [_t(d) for d in dys]
    c = xs[0].shape[1]
    i64 = dict(dtype=torch.int64, device=DEV)

    def each(fn, *shape):
        outs = [torch.full(shape, -7, **i64) for _ in xs]
        for k, x in enumerate(xs):
            fn(k, x, outs[k])
        return outs

    mw = torch.stack(each(lambda k, x, o: h.sync_bn_max(x, o), 2 * c)).amax(0)
    sw = torch.stack(each(lambda k, x, o: h.sync_bn_sum(x, mw, o), 2 * c + 1)).sum(0)
    mean = torch.empty(c, dtype=torch.float64, device=DEV)
    qw = torch.stack(each(lambda k, x, o: h.sync_bn_sumsq(x, mw, sw, mean, o), 4 * c)).sum(0)
    var, invstd = torch.empty_like(mean), torch.empty_like(mean)
    g, b = _t(gamma), _t(beta)
    rmt, rvt = _t(rm), _t(rv)
    ys = []
    for k, x in enumerate(xs):
        y = torch.empty_like(x)
        # the running statistics are updated once (by "rank" 0 here; every rank computes the same bits)
        h.sync_bn_apply(x, mw, sw, mean, qw, g, b, eps, momentum, rmt if k == 0 else None, rvt if k == 0 else None, var, invstd, y)
        ys.append(y)
    bmw = torch.stack(each(lambda k, x, o: h.sync_bn_backward_max(dys[k], x, mean, invstd, o), 3 * c)).amax(0)
    dgs = [torch.empty(c, device=DEV) for _ in xs]
    dbs = [torch.empty(c, device=DEV) for _ in xs]
    loc = each(lambda k, x, o: h.sync_bn_backward_sum(dys[k], x, mean, invstd, bmw, o, dgs[k], dbs[k]), 4 * c)
    bsw = torch.stack(loc).sum(0)
    dxs = []
    for k, x in enumerate(xs):
        dx = torch.empty_like(x)
        h.sync_bn_backward_apply(dys[k], x, mean, invstd, g, bmw, bsw, sw[2 * c:], dx)
        dxs.append(dx)
    torch.cuda.synchronize()
    np_ = lambda t: t.cpu().numpy()  # noqa: E731
    return {"max_words": np_(mw), "sum_words": np_(sw), "sq_words": np_(qw), "mean": np_(mean), "var": np_(var), "invstd": np_(invstd),
            "ys": [np_(y) for y in ys], "bmax_words": np_(bmw), "bsum_words": np_(bsw), "dgammas": [np_(d) for d in dgs],
            "dbetas": [np_(d) for d in dbs], "dxs": [np_(d) for d in dxs],
            "running_mean": None if rmt is None else np_(rmt), "running_var": None if rvt is None else np_(rvt)}


def reference(xs, dys, gamma, beta, eps=1e-5, momentum=0.1, rm=None, rv=None):
    f = R.forward(xs, gamma, beta, eps, momentum, rm, rv)
    b = R.backward(dys, xs, f, gamma)
    mean, invstd = f["mean"], f["invstd"]
    bmw = R.combine_max([R.bwd_max(d, x, mean, invstd) for d, x in zip(dys, xs)])
    bsw = R.combine_sum([R.bwd_sum(d, x, mean, invstd, bmw)[0] for d, x in zip(dys, xs)])
    return {**f, **b, "bmax_words": bmw, "bsum_words": bsw}


def bits(a):
    """the bytes of `a` with every NaN made the same NaN (the payload and sign of a NaN are not part of the contract)"""
    a = np.array(a)
    if a.dtype.kind == "f":
        a[np.isnan(a)] = np.nan
    return a.tobytes()


def assert_same_bits(got, ref):
    for k in ("max_words", "sum_words", "sq_words", "mean", "var", "invstd", "bmax_words", "bsum_words", "running_mean", "running_var"):
        if ref.get(k) is None:
            continue
        assert bits(got[k]) == bits(ref[k]), k
    for k in ("ys", "dxs", "dgammas", "dbetas"):
        for r, (a, b) in enumerate(zip(got[k], ref[k])):
            assert bits(a) == bits(b), (k, r, np.argwhere((a != b) & ~(np.isnan(a) & np.isnan(b)))[:5])


def problem(n, c, seed, edge=True):
    g = np.random.default_rng(seed)
    x = (g.standard_normal((n, c), dtype=np.float32) * g.uniform(0.01, 10, c).astype(np.float32)
         + g.uniform(-5, 5, c).astype(np.float32))
    dy = g.standard_normal((n, c), dtype=np.float32)
    if edge and c >= 8:
        x[:, 0] = 2.5                                                  # constant channel
        x[:, 1] = (g.standard_normal(n) * 1e-3).astype(np.float32)     # outlier channel: sigma 1e-3, max 1e4
        x[n // 3, 1] = 1e4
        x[:, 2] = (g.standard_normal(n) * 1e-40).astype(np.float32)    # subnormals
        x[n // 2, 3] = np.nan
        x[n // 5, 4] = np.inf
        x[n - 1, 5] = -np.inf
        dy[n // 7, 6] = np.nan
        dy[n // 4, 7] = -np.inf
    gamma = g.uniform(0.5, 2, c).astype(np.float32)
    beta = g.uniform(-1, 1, c).astype(np.float32)
    return x, dy, gamma, beta


WIDTHS = [32, 64, 96, 128, 256]


@pytest.mark.gpu
@pytest.mark.parametrize("c", WIDTHS)
@pytest.mark.parametrize("n", [1, 2, 1000, 65_537])
def test_kernels_match_the_restatement(c, n):
    x, dy, gamma, beta = problem(n, c, seed=c + n)
    rm, rv = np.linspace(-1, 1, c).astype(np.float32), np.linspace(0.5, 2, c).astype(np.float32)
    got = gpu_pass([x], [dy], gamma, beta, 1e-5, 0.1, rm, rv)
    ref = reference([x], [dy], gamma, beta, 1e-5, 0.1, rm, rv)
    assert_same_bits(got, ref)
    if n > 10:
        assert np.isnan(got["ys"][0][:, 3:6]).all() and np.isnan(got["dxs"][0][:, 3:8]).all()
        assert np.isfinite(got["ys"][0][:, :3]).all() and np.isfinite(got["dxs"][0][:, :3]).all()
        assert np.isfinite(got["dxs"][0][:, 8:]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n,c", [(1_048_576, 128), (2_000_003, 64), (4_194_304, 32)], ids=["1M-128", "2M-64", "4M-32"])
def test_kernels_match_the_restatement_at_millions_of_rows(n, c):
    x, dy, gamma, beta = problem(n, c, seed=n % 1000)
    got = gpu_pass([x], [dy], gamma, beta)
    assert_same_bits(got, reference([x], [dy], gamma, beta))
    again = gpu_pass([x], [dy], gamma, beta)
    assert_same_bits(again, got)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [64, 256])
def test_bits_do_not_depend_on_row_order_or_the_split(c):
    n = 30_001
    x, dy, gamma, beta = problem(n, c, seed=5)
    one = gpu_pass([x], [dy], gamma, beta)
    for world, seed in ((2, 1), (3, 2), (4, 3)):
        perm, idx = fake.split_rows(n, world, seed)
        got = gpu_pass([x[i] for i in idx], [dy[i] for i in idx], gamma, beta)
        for k in ("mean", "var", "invstd", "max_words", "sum_words", "sq_words", "bmax_words", "bsum_words"):
            assert bits(got[k]) == bits(one[k]), (world, k)
        for k in ("ys", "dxs"):
            assert bits(sync_bn_ranks.rows_of(got[k], perm, n)) == bits(one[k][0]), (world, k)


@pytest.mark.gpu
def test_empty_rank_takes_part():
    x, dy, gamma, beta = problem(500, 64, seed=9)
    got = gpu_pass([x, x[:0]], [dy, dy[:0]], gamma, beta)
    assert_same_bits({**got, "ys": got["ys"][:1], "dxs": got["dxs"][:1], "dgammas": got["dgammas"][:1], "dbetas": got["dbetas"][:1]},
                     reference([x], [dy], gamma, beta))
    assert (got["dgammas"][1][8:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2])
def test_two_processes_on_one_gpu_give_the_bits_of_one_process(tmp_path, world):
    n, c = 20_011, 128
    x, dy, gamma, beta = problem(n, c, seed=21, edge=False)
    perm, idx = fake.split_rows(n, world, seed=4)
    res = fake.run_ranks(sync_bn_ranks.bn_rank, world, tmp_path, [x[i] for i in idx], [dy[i] for i in idx], gamma, beta, DEV,
                         fake=False, timeout=600)
    one = gpu_pass([x], [dy], gamma, beta, 1e-5, 0.1, np.zeros(c, np.float32), np.ones(c, np.float32))
    assert sync_bn_ranks.rows_of([r["y"] for r in res], perm, n).tobytes() == one["ys"][0].tobytes()
    assert sync_bn_ranks.rows_of([r["dx"] for r in res], perm, n).tobytes() == one["dxs"][0].tobytes()
    for r in res:
        for k in ("mean", "var", "invstd", "running_mean", "running_var"):
            assert r[k].tobytes() == one[k].tobytes(), k


def test_sync_bn_kernels_have_no_stack_frame_and_no_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "lidiff_b200", "csrc", "sync_bn.cu"), "-o", str(tmp_path / "sync_bn.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    found = re.findall(r"Function properties for (\S*sbn\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    assert len(found) == 10, log
    for name, *counts in found:
        assert counts == ["0", "0", "0"], (name, counts)


@pytest.mark.gpu
def test_a_combined_row_count_of_2_31_or_more_gives_nan():
    """the words are exact for fewer than 2^31 rows in all: a larger combined count (only seen on the device) gives NaN statistics,
    outputs and running statistics rather than wrapped sums"""
    h = _lib.get_handle(DEV)
    x, dy, gamma, beta = (_t(a) for a in problem(1000, 32, seed=3, edge=False))
    c = 32
    i64 = dict(dtype=torch.int64, device=DEV)
    mw, sw, qw, bmw, bsw = (torch.empty(k, **i64) for k in (2 * c, 2 * c + 1, 4 * c, 3 * c, 4 * c))
    mean, var, invstd = (torch.empty(c, dtype=torch.float64, device=DEV) for _ in range(3))
    rm, rv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    y, dx = torch.empty_like(x), torch.empty_like(x)
    h.sync_bn_max(x, mw)
    h.sync_bn_sum(x, mw, sw)
    sw[2 * c] += 1 << 31                                 # as if other ranks had contributed 2^31 rows
    h.sync_bn_sumsq(x, mw, sw, mean, qw)
    h.sync_bn_apply(x, mw, sw, mean, qw, gamma, beta, 1e-5, 0.1, rm, rv, var, invstd, y)
    for t in (mean, var, invstd, y, rm, rv):
        assert torch.isnan(t).all()
    # the backward with a valid forward and an out-of-range count
    sw[2 * c] -= 1 << 31
    h.sync_bn_sumsq(x, mw, sw, mean, qw)
    h.sync_bn_apply(x, mw, sw, mean, qw, gamma, beta, 1e-5, 0.1, None, None, var, invstd, y)
    assert torch.isfinite(y).all()
    h.sync_bn_backward_max(dy, x, mean, invstd, bmw)
    h.sync_bn_backward_sum(dy, x, mean, invstd, bmw, bsw, None, None)
    h.sync_bn_backward_apply(dy, x, mean, invstd, gamma, bmw, bsw, sw[2 * c:] + (1 << 31), dx)
    assert torch.isnan(dx).all()
