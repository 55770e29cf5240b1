"""TEST INFRASTRUCTURE: CPU stand-ins for the seven lb2_sync_bn_* entry points (the restatement in tests/sync_bn_reference.py) on top
of the diffusion-training fake, and a runner that starts gloo ranks as processes, so that the synchronised batch norm's host logic
(the autograd wiring, the collectives between the calls, the CLIs' data-parallel steps) runs without a GPU."""
import os
import time
import traceback

import numpy as np
import torch

import fake_diffusion_backend
import sync_bn_reference as R
from lidiff_b200 import _lib


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


class FakeSyncBNHandle(fake_diffusion_backend.FakeDiffusionHandle):
    def sync_bn_max(self, x, max_words):
        max_words.copy_(torch.from_numpy(R.fwd_max(_np(x))))

    def sync_bn_sum(self, x, max_words, sum_words):
        sum_words.copy_(torch.from_numpy(R.fwd_sum(_np(x), _np(max_words))))

    def sync_bn_sumsq(self, x, max_words, sum_words, mean, sq_words):
        m, w = R.fwd_sumsq(_np(x), _np(max_words), _np(sum_words))
        mean.copy_(torch.from_numpy(m))
        sq_words.copy_(torch.from_numpy(w))

    def sync_bn_apply(self, x, max_words, sum_words, mean, sq_words, gamma, beta, eps, momentum, running_mean, running_var, var, invstd,
                      y):
        v, i, yy, rm, rv = R.fwd_apply(_np(x), _np(max_words), _np(sum_words), _np(mean), _np(sq_words), _np(gamma), _np(beta), eps,
                                       momentum, _np(running_mean), _np(running_var))
        var.copy_(torch.from_numpy(v))
        invstd.copy_(torch.from_numpy(i))
        y.copy_(torch.from_numpy(yy))
        if running_mean is not None:
            running_mean.copy_(torch.from_numpy(rm))
            running_var.copy_(torch.from_numpy(rv))

    def sync_bn_backward_max(self, dy, x, mean, invstd, max_words):
        max_words.copy_(torch.from_numpy(R.bwd_max(_np(dy), _np(x), _np(mean), _np(invstd))))

    def sync_bn_backward_sum(self, dy, x, mean, invstd, max_words, sum_words, dgamma, dbeta):
        w, dg, db = R.bwd_sum(_np(dy), _np(x), _np(mean), _np(invstd), _np(max_words))
        sum_words.copy_(torch.from_numpy(w))
        if dgamma is not None:
            dgamma.copy_(torch.from_numpy(dg))
        if dbeta is not None:
            dbeta.copy_(torch.from_numpy(db))

    def sync_bn_backward_apply(self, dy, x, mean, invstd, gamma, max_words, sum_words, count, dx):
        dx.copy_(torch.from_numpy(R.bwd_apply(_np(dy), _np(x), _np(mean), _np(invstd), _np(gamma), _np(max_words), _np(sum_words),
                                              int(count[0]))))


def install_plain():
    """install() without pytest's monkeypatch, for rank processes; returns the handle"""
    from lidiff_b200 import me
    h = FakeSyncBNHandle()
    h.emulate_tc = True
    _lib.get_handle = lambda device=None: h
    me._require_cuda = lambda t, what: None
    return h


def install(monkeypatch):
    from lidiff_b200 import me
    h = FakeSyncBNHandle()
    h.emulate_tc = True
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    monkeypatch.setattr(me, "_require_cuda", lambda t, what: None)
    return h


def _rank_main(rank, fn, world, tmp, args, fake):
    import torch.distributed as dist
    try:
        if fake:
            install_plain()
        dist.init_process_group("gloo", init_method=f"file://{os.path.join(tmp, 'rendezvous')}", rank=rank, world_size=world)
        try:
            out = fn(rank, world, *args)
        finally:
            dist.destroy_process_group()
        torch.save(out, os.path.join(tmp, f"rank{rank}.pt"))
    except Exception:
        with open(os.path.join(tmp, f"rank{rank}.err"), "w") as f:
            f.write(traceback.format_exc())
        raise


def run_ranks(fn, world, tmp, *args, fake=True, timeout=600):
    """fn(rank, world, *args) in `world` gloo processes (fn importable by name); returns the ranks' results in rank order"""
    import torch.multiprocessing as mp
    tmp = str(tmp)
    os.makedirs(tmp, exist_ok=True)
    ctx = mp.start_processes(_rank_main, args=(fn, world, tmp, args, fake), nprocs=world, join=False, start_method="spawn")
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=max(1.0, deadline - time.monotonic())):       # join returns after each process that ends
            if time.monotonic() > deadline:
                raise AssertionError(f"the ranks did not finish within {timeout} s")
    except Exception:
        errs = [open(os.path.join(tmp, f)).read() for f in sorted(os.listdir(tmp)) if f.endswith(".err")]
        raise AssertionError("\n".join(errs) or "a rank failed")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
                p.join(10)
            if p.is_alive():
                p.kill()
            p.join()
    return [torch.load(os.path.join(tmp, f"rank{r}.pt"), weights_only=False) for r in range(world)]


def split_rows(n, world, seed):
    """a shuffled, uneven split of range(n) into `world` parts: (perm, list of index arrays)"""
    g = np.random.default_rng(seed)
    perm = g.permutation(n)
    cuts = np.sort(g.choice(np.arange(1, n), world - 1, replace=False))
    return perm, np.split(perm, cuts)
