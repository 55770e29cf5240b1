"""TEST INFRASTRUCTURE: CPU stand-ins for lb2_spconv_wgrad and lb2_segment_sum (fp64 restatements of include/lidiff_b200.h) on top
of the refinement fake, so that the training path's host logic (autograd wiring, adjoint maps and weight transforms, checkpoints)
runs without a GPU.  Tests install it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_refine_backend
from lidiff_b200 import _lib


def restate_wgrad(x, g, nbr, kvol):
    """dw[k] = sum over o with nbr[k][o] >= 0 of x[nbr[k][o]]^T g[o], fp64 (nbr None: identity)"""
    x, g = x.double(), g.double()
    dw = torch.zeros(kvol, x.shape[1], g.shape[1], dtype=torch.float64)
    for k in range(kvol):
        src = torch.arange(g.shape[0]) if nbr is None else nbr[k, : g.shape[0]].long()
        o = torch.nonzero(src >= 0)[:, 0]
        dw[k] = x[src[o]].T @ g[o]
    return dw


class FakeTrainHandle(fake_refine_backend.FakeRefineHandle):
    def spconv_wgrad(self, x, g, nbr, kvol, dw):
        self.launches += 3
        dw.copy_(restate_wgrad(x, g, nbr, kvol).to(dw.dtype))

    def segment_sum(self, values, order, offsets, out):
        self.launches += 1
        v = values if order is None else values[order]
        for s in range(offsets.shape[0] - 1):
            acc = torch.zeros(values.shape[1], dtype=values.dtype)
            for i in range(int(offsets[s]), int(offsets[s + 1])):
                acc = acc + v[i]
            out[s] = acc


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake and let the ME surface take CPU tensors; returns the handle"""
    from lidiff_b200 import me
    h = FakeTrainHandle()
    h.emulate_tc = True
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    monkeypatch.setattr(me, "_require_cuda", lambda t, what: None)
    return h
