"""CPU fakes of the device random streams (lb2_mt19937_words, lb2_legacy_gauss, lb2_randperm) from the numpy restatements in
rng_reference.py, added to the refinement and diffusion sample fakes, so the host logic of device_rng=True runs without a GPU."""
import numpy as np
import torch

import fake_refine_backend
import fake_samples_backend
import rng_reference as R
from lidiff_b200 import _lib


class FakeRngMixin:
    def mt19937_words(self, state, pos, n, out):
        words, key, pos2 = R.mt_words(state.numpy().view(np.uint32), pos, n)
        out[:n] = torch.from_numpy(words.view(np.int32))
        state[:] = torch.from_numpy(key.view(np.int32))
        return pos2

    def legacy_gauss(self, words, n_words, n_out, has_gauss, gauss, band, out):
        """lb2_legacy_gauss' contract: logs within the band from libm, the rest the correct rounding (a long-double log)"""
        hg = 1 if has_gauss else 0
        if n_out == 0:
            return _lib.GaussInfo(0, 0, 0, hg, gauss)
        if hg:
            out[0] = gauss
        pairs = (n_out - hg + 1) // 2
        if pairs == 0:
            return _lib.GaussInfo(0, 0, 0, 0, 0.0)
        x1, x2, r2, acc = R.attempts(words[:n_words].numpy().view(np.uint32))
        if acc.sum() < pairs:
            return _lib.GaussInfo(0, 0, 1, hg, gauss)
        ks = np.flatnonzero(acc)[:pairs]
        r2k = r2[ks]
        host = R.deferred(r2k, band)
        logs = np.log(r2k.astype(np.longdouble)).astype(np.float64)
        logs[host] = R.libm_log(r2k[host])
        f = np.sqrt(-2.0 * logs / r2k)
        o = hg + 2 * np.arange(pairs)
        res = out[:n_out].numpy()
        res[o] = f * x2[ks]
        last = o + 1 < n_out
        res[o[last] + 1] = (f * x1[ks])[last]
        odd = (n_out - hg) % 2 == 1
        return _lib.GaussInfo(4 * (int(ks[-1]) + 1), int(host.sum()), 0, int(odd), float(f[-1] * x1[ks[-1]]) if odd else 0.0)

    def randperm(self, words, n, out, d_rounds=None):
        w = words.numpy().view(np.uint32) if words is not None else np.zeros(0, np.uint32)
        perm, rounds = R.randperm_rounds(w, n)
        out[:] = torch.from_numpy(perm)
        if d_rounds is not None:
            d_rounds.fill_(rounds)


class FakeRefineRngHandle(FakeRngMixin, fake_refine_backend.FakeRefineHandle):
    pass


class FakeSamplesRngHandle(FakeRngMixin, fake_samples_backend.FakeSamplesHandle):
    pass


def install_refine(monkeypatch):
    h = FakeRefineRngHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h


def install_samples(monkeypatch):
    fake_samples_backend.install(monkeypatch)
    h = FakeSamplesRngHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
