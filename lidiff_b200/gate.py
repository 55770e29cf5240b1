"""The conditioning gate's multiply-gather with its gradients: out = x * table[idx].

Every voxel row is scaled by the row of `table` that its nearest part voxel selects, so a few thousand table rows serve 10^5 - 10^6
voxel rows, and in the unconditional training step one table row per scan serves them all.  The gradients are
    d x     = G * table[idx]                                    (lb2_gate_mul, the forward's kernel)
    d table = sum over the rows with idx = j of G * x            (lb2_segment_dot: chunks of the sorted rows, no atomics)
so neither the gathered table nor the product G * x is ever materialised, and two backward passes give the same bits."""
from __future__ import annotations

import torch

from . import _lib


def index_dot(a: torch.Tensor, b: torch.Tensor | None, idx: torch.Tensor, n: int) -> torch.Tensor:
    """(n, c) fp32: row j = sum of a[i] * b[i] (b None: of a[i]) over the rows i with idx[i] == j, in lb2_segment_dot's order over
    the rows sorted stably by idx; a, b (len(idx), c) fp32"""
    a = a.contiguous()
    b = None if b is None else b.contiguous()
    out = torch.empty((n, a.shape[1]), dtype=a.dtype, device=a.device)
    idx = idx.long()
    order = torch.sort(idx, stable=True).indices
    offsets = torch.zeros(n + 1, dtype=torch.int64, device=a.device)
    torch.cumsum(torch.bincount(idx, minlength=n), 0, out=offsets[1:])
    _lib.get_handle(a.device).segment_dot(a, b, order, offsets, out)
    return out


def _mul_rows(x, table, idx32):
    out = torch.empty_like(x)
    if x.shape[0] > 0:
        _lib.get_handle(x.device).gate_mul(x, table, idx32, None, x.shape[0], x.shape[1], out)
    return out


class GateMul(torch.autograd.Function):
    """out = x * table[idx]; x (M, C) fp32, table (M_part, C) fp32, idx (M) integer rows of table"""

    @staticmethod
    def forward(ctx, x, table, idx):
        x, table, idx32 = x.contiguous(), table.contiguous(), idx.to(torch.int32).contiguous()
        ctx.save_for_backward(x, table, idx32)
        return _mul_rows(x, table, idx32)

    @staticmethod
    def backward(ctx, G):
        x, table, idx32 = ctx.saved_tensors
        G = G.contiguous()
        dx = _mul_rows(G, table, idx32) if ctx.needs_input_grad[0] else None
        dtable = index_dot(G, x, idx32, table.shape[0]) if ctx.needs_input_grad[1] else None
        return dx, dtable, None


class TakeRows(torch.autograd.Function):
    """y = src[idx] (the time embedding of every part row's batch); backward: index_dot of the gradient alone, so that a batch's
    thousands of part rows are summed by chunks and in a fixed order"""

    @staticmethod
    def forward(ctx, src, idx):
        ctx.save_for_backward(idx)
        ctx.n = src.shape[0]
        return src[idx]

    @staticmethod
    def backward(ctx, grad):
        (idx,) = ctx.saved_tensors
        return index_dot(grad, None, idx, ctx.n), None
