"""The tensor-core convolution loads a row's neighbour indices only for the offsets its row mask names.  An exact mask, no mask
(every offset loaded) and an all-ones mask give the same bits, for both passes and both channel halves of a Cout-256 layer."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def random_field(n, spread, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(n, 3, generator=g) * spread
    return torch.cat([torch.zeros(n, 1), torch.round(pts / 0.05)], 1)


@pytest.mark.parametrize("c1,c2,cout,lvl,kind", [(32, 0, 32, 0, "3"), (96, 32, 96, 1, "3"), (256, 128, 256, 3, "3"),
                                                    (256, 0, 256, 3, "up"), (32, 0, 64, 2, "dn")])
def test_row_mask_skips_only_absent_offsets(c1, c2, cout, lvl, kind):
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    from lidiff_b200.engine import Geometry
    h = _lib.get_handle(DEV)
    coords = random_field(70_000, 1.0 if lvl >= 3 else 0.3, 43)
    N = coords.shape[0]
    g = Geometry(h, N)
    g.build(coords.to(DEV).contiguous(), N)
    M = g.sizes()[lvl]
    nbr, perm, kvol = {"3": (g.nbr3[lvl], g.perm3[lvl], 27), "up": (g.nbr_up[lvl], g.perm_up[lvl], 8),
                       "dn": (g.nbr_dn[lvl], g.perm_dn[lvl], 8)}[kind]
    exact = g.mask_of[nbr.data_ptr()]
    ones = torch.full_like(exact, (1 << kvol) - 1)
    gen = torch.Generator().manual_seed(c1 + cout + lvl)
    W = (torch.randn(kvol, c1 + c2, cout, generator=gen) / np.sqrt((c1 + c2) * kvol)).to(DEV)
    Wp = h.pack_weights(W)
    A = torch.randn(2, N, c1, generator=gen).to(DEV)
    B = torch.randn(2, N, c2, generator=gen).to(DEV) if c2 else None
    R = torch.randn(2, N, cout, generator=gen).to(DEV)
    res = []
    for mask in (None, exact, ones):
        out = torch.full((2, N, cout), float("nan"), device=DEV)
        d = ConvDesc()
        d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, kvol
        d.weight, d.weight_packed, d.relu = W.data_ptr(), Wp.data_ptr(), 1
        d.nbr, d.nbr_stride, d.d_mout, d.mout_cap, d.npass = nbr.data_ptr(), N, g.d_n[lvl].data_ptr(), N, 2
        d.row_perm = perm.data_ptr()
        d.row_mask = mask.data_ptr() if mask is not None else None
        d.tile_order128 = g.tile_order_of[nbr.data_ptr()][0].data_ptr()
        for p_ in range(2):
            d.io[p_] = ConvIO(A[p_].data_ptr(), B[p_].data_ptr() if B is not None else None, R[p_].data_ptr(), out[p_].data_ptr(),
                              None, None, None)
        h.spconv(d, _lib.ALGO_TC)
        torch.cuda.synchronize()
        res.append(out[:, :M].clone())
    assert not torch.isnan(res[0]).any(), "a live row was not written"
    assert res[0].abs().sum() > 0
    for r in res[1:]:
        assert torch.equal(res[0], r)
