"""TEST INFRASTRUCTURE: the training fake (tests/fake_train_backend.py) with a CPU stand-in for lb2_segment_dot, so that the host logic
of diffusion training (the hoisted gates, the training step, checkpoints) runs without a GPU.  fp32 operands go through the kernel's
documented order (tests/segment_dot_reference.py); fp64 operands, which the library does not take, are summed by torch so that the
gate's autograd wiring can be checked in double precision."""
import torch

import fake_train_backend
import segment_dot_reference as sdr
from lidiff_b200 import _lib


class FakeDiffusionHandle(fake_train_backend.FakeTrainHandle):
    def segment_dot(self, a, b, order, offsets, out):
        self.launches += 2
        if a.dtype == torch.float32:
            out.copy_(torch.from_numpy(sdr.emulate(a.detach().numpy(), None if b is None else b.detach().numpy(),
                                                   None if order is None else order.numpy(), offsets.numpy())))
            return
        p = a if b is None else a * b
        p = p if order is None else p[order]
        for s in range(offsets.shape[0] - 1):
            out[s] = p[int(offsets[s]): int(offsets[s + 1])].sum(0)


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake and let the ME surface take CPU tensors; returns the handle"""
    from lidiff_b200 import me
    h = FakeDiffusionHandle()
    h.emulate_tc = True
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    monkeypatch.setattr(me, "_require_cuda", lambda t, what: None)
    return h
