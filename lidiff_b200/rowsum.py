"""Deterministic backward of a row gather: out[j] = sum of values[i] over the rows i with idx[i] == j, added in ascending i.

The gather y = src[idx] has the gradient d src[j] = sum_{idx[i] = j} dy[i].  An atomic scatter-add (index_add_ / index_put_ with
accumulate on CUDA) adds in whatever order the threads arrive, so two backward passes differ in the last bits.  Here the rows are
grouped by a stable sort of idx and each group is summed in row order by one kernel (lb2_segment_sum), so the result depends on
the inputs only."""
from __future__ import annotations

import torch

from . import _lib


def index_sum(values: torch.Tensor, idx: torch.Tensor, n: int) -> torch.Tensor:
    """(n, c) tensor of values' dtype: row j = sum of values[i] over i with idx[i] == j, in ascending i; values (len(idx), c)"""
    values = values.contiguous()
    out = torch.empty((n, values.shape[1]), dtype=values.dtype, device=values.device)
    if n == 0:
        return out
    if values.shape[0] == 0:            # no rows: every sum is empty (and an empty tensor has no data pointer to pass)
        return out.zero_()
    idx = idx.long()
    order = torch.sort(idx, stable=True).indices
    offsets = torch.zeros(n + 1, dtype=torch.int64, device=values.device)
    torch.cumsum(torch.bincount(idx, minlength=n), 0, out=offsets[1:])
    _lib.get_handle(values.device).segment_sum(values, order, offsets, out)
    return out


class GatherRows(torch.autograd.Function):
    """y = src[idx] with index_sum as its backward (the forward is torch's indexing, so its values are those of src[idx])"""

    @staticmethod
    def forward(ctx, src, idx):
        ctx.save_for_backward(idx)
        ctx.n = src.shape[0]
        return src[idx]

    @staticmethod
    def backward(ctx, grad):
        (idx,) = ctx.saved_tensors
        return index_sum(grad, idx, ctx.n), None
