"""The tensor-core convolution is persistent: each CTA runs a strided sequence of (tile, pass, channel half) work items through one
stage ring.  These tests check that a CTA's items do not see each other's state: any dispatch order gives the same bits, tiles
without neighbours between live ones give the epilogue of a zero sum, the two passes may gather by different paths, and the live
row count (down to one row, and fewer live items than SMs) decides exactly which rows are written."""
import numpy as np
import pytest
import torch

from oracle import me_cpu as ome

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def random_field(n, spread, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(n, 3, generator=g) * spread
    return torch.cat([torch.zeros(n, 1), torch.round(pts / 0.05)], 1)


def rel_err(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs() / (b.abs() + b.pow(2).mean().sqrt() + 1e-30)).max().item()


def split_of(h, x):
    """fp16 hi/lo companion of x (npass, n, c) through the library's own split (gate_mul by 1)."""
    n, c = x.shape[1], x.shape[2]
    one = torch.ones(1, c, device=DEV)
    xh = torch.zeros(x.shape[0], n, 2 * c, dtype=torch.float16, device=DEV)
    for p_ in range(x.shape[0]):
        h.gate_mul(x[p_], one, None, None, n, c, torch.empty_like(x[p_]), xh[p_])
    return xh


def conv(h, W, Wp, A, B, R, sc_, sh_, nbr, n, d_mout, perm=None, mask=None, order=None, A_h=None, B_h=None):
    """One ALGO_TC launch over two passes into a NaN-filled output; io[p].in1_h / in2_h are set where A_h[p] / B_h[p] is given."""
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    kvol, cin, cout = W.shape
    c1 = A.shape[-1]
    out = torch.full((2, n, cout), float("nan"), device=DEV)
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = c1, cin - c1, cout, kvol
    d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
    d.scale, d.shift, d.relu = sc_.data_ptr(), sh_.data_ptr(), 1
    d.nbr = nbr.data_ptr() if nbr is not None else None
    d.nbr_stride, d.d_mout, d.mout_cap, d.npass = n, d_mout.data_ptr(), n, 2
    d.row_perm = perm.data_ptr() if perm is not None else None
    d.row_mask = mask.data_ptr() if mask is not None else None
    d.tile_order128 = order.data_ptr() if order is not None else None
    ptr = lambda t, p_: t[p_].data_ptr() if t is not None and t[p_] is not None else None
    for p_ in range(2):
        d.io[p_] = ConvIO(A[p_].data_ptr(), ptr(B, p_), R[p_].data_ptr(), out[p_].data_ptr(), None, None, None, None,
                          ptr(A_h, p_), ptr(B_h, p_), None, None, None)
    h.spconv(d, _lib.ALGO_TC)
    torch.cuda.synchronize()
    return out


def operands(kvol, c1, c2, cout, n, seed):
    gen = torch.Generator().manual_seed(seed)
    W = (torch.randn(kvol, c1 + c2, cout, generator=gen) / np.sqrt((c1 + c2) * kvol)).to(DEV)
    A = torch.randn(2, n, c1, generator=gen).to(DEV)
    B = torch.randn(2, n, c2, generator=gen).to(DEV) if c2 else None
    R = torch.randn(2, n, cout, generator=gen).to(DEV)
    sc_, sh_ = (torch.rand(cout, generator=gen) + 0.5).to(DEV), torch.randn(cout, generator=gen).to(DEV)
    return W, A, B, R, sc_, sh_


@pytest.fixture(scope="module")
def geo():
    from lidiff_b200 import _lib
    from lidiff_b200.engine import Geometry
    h = _lib.get_handle(DEV)
    coords = random_field(70_000, 3.0, 47)        # 7k - 68k rows on levels 1-4: several work items per CTA
    n = coords.shape[0]
    g = Geometry(h, n)
    g.build(coords.to(DEV).contiguous(), n)
    return dict(h=h, g=g, n=n, coords=coords)


@pytest.mark.parametrize("c1,c2,cout,lvl,kind", [(96, 32, 96, 1, "3"), (256, 128, 256, 3, "3"), (256, 0, 256, 3, "up"),
                                                    (32, 0, 64, 2, "dn"), (64, 0, 128, 1, "1")])
def test_any_dispatch_order_gives_the_same_bits(geo, c1, c2, cout, lvl, kind):
    h, g, n = geo["h"], geo["g"], geo["n"]
    M = g.sizes()[lvl]
    nbr, perm, kvol = {"3": (g.nbr3[lvl], g.perm3[lvl], 27), "up": (g.nbr_up[lvl], g.perm_up[lvl], 8),
                       "dn": (g.nbr_dn[lvl], g.perm_dn[lvl], 8), "1": (None, None, 1)}[kind]
    W, A, B, R, sc_, sh_ = operands(kvol, c1, c2, cout, n, c1 + cout + lvl)
    Wp = h.pack_weights(W)
    nt = (M + 127) // 128
    assert nt * 2 * (2 if cout > 128 else 1) > 2 * torch.cuda.get_device_properties(DEV).multi_processor_count, "too few items per CTA"
    if nbr is None:                              # 1x1: natural order only, checked against fp64
        out = conv(h, W, Wp, A, B, R, sc_, sh_, None, n, g.d_n[lvl])
        for p_ in range(2):
            y = torch.relu((A[p_][:M].double() @ W[0].double()) * sc_.double() + sh_.double() + R[p_][:M].double())
            assert rel_err(out[p_][:M], y) < 5e-5
        assert torch.isnan(out[:, M:]).all()
        return
    mask = g.mask_of[nbr.data_ptr()]
    order = g.tile_order_of[nbr.data_ptr()][0]
    res = []
    for seed in range(3):
        o = order.clone()
        if seed:                                 # a random permutation of the live tiles
            o[:nt] = o[:nt][torch.randperm(nt, generator=torch.Generator().manual_seed(seed)).to(DEV)]
        res.append(conv(h, W, Wp, A, B, R, sc_, sh_, nbr, n, g.d_n[lvl], perm, mask, o)[:, :M])
    assert not torch.isnan(res[0]).any(), "a live tile was not run"
    assert res[0].abs().sum() > 0
    for r in res[1:]:
        assert torch.equal(res[0], r)


@pytest.mark.parametrize("cin,cout", [(64, 64), (128, 256)])
def test_tiles_without_neighbours_between_live_tiles(cin, cout):
    """Whole tiles whose rows have no neighbour (every 5th tile, natural order) run only the epilogue of a zero sum."""
    from lidiff_b200 import _lib
    h = _lib.get_handle(DEV)
    n, kvol = 64_000, 27                         # 500 tiles: several items per CTA, empty ones between live ones
    gen = torch.Generator().manual_seed(cin + cout)
    have = torch.rand(kvol, n, generator=gen) < 0.3
    nbr = torch.where(have, torch.randint(0, n, (kvol, n), generator=gen, dtype=torch.int32), torch.tensor(-1, dtype=torch.int32))
    empty_rows = ((torch.arange(n) // 128) % 5 == 2)
    holed = nbr.clone()
    holed[:, empty_rows] = -1
    mask_of = lambda m: ((m >= 0).int() << torch.arange(kvol, dtype=torch.int32)[:, None]).sum(0, dtype=torch.int32)
    W, A, _, R, sc_, sh_ = operands(kvol, cin, 0, cout, n, 5)
    Wp = h.pack_weights(W)
    d_n = torch.tensor([n], dtype=torch.int32, device=DEV)
    full = conv(h, W, Wp, A, None, R, sc_, sh_, nbr.to(DEV), n, d_n, mask=mask_of(nbr).to(DEV))
    out = conv(h, W, Wp, A, None, R, sc_, sh_, holed.to(DEV), n, d_n, mask=mask_of(holed).to(DEV))
    e = empty_rows.to(DEV)
    assert torch.equal(out[:, ~e], full[:, ~e]), "live rows changed"
    assert torch.equal(out[:, e], torch.relu(sh_ + R[:, e])), "an empty tile is not the epilogue of a zero sum"


@pytest.mark.parametrize("c1,c2,cout,lvl", [(64, 32, 64, 2), (128, 0, 256, 3)])
def test_passes_may_gather_by_different_paths(geo, c1, c2, cout, lvl):
    """Pass 0 gathers the fp16 split companions with cp.async, pass 1 the fp32 rows: each pass gives the bits of a launch in which
    both passes take its path."""
    h, g, n = geo["h"], geo["g"], geo["n"]
    nbr, perm = g.nbr3[lvl], g.perm3[lvl]
    M = g.sizes()[lvl]
    W, A, B, R, sc_, sh_ = operands(27, c1, c2, cout, n, c1 + c2 + cout)
    Wp = h.pack_weights(W)
    A_h = split_of(h, A)
    B_h = split_of(h, B) if B is not None else None
    args = (h, W, Wp, A, B, R, sc_, sh_, nbr, n, g.d_n[lvl], perm, g.mask_of[nbr.data_ptr()], g.tile_order_of[nbr.data_ptr()][0])
    companions = conv(*args, A_h=A_h, B_h=B_h)
    fp32 = conv(*args)
    mixed = conv(*args, A_h=[A_h[0], None], B_h=[B_h[0], None] if B_h is not None else None)
    assert not torch.isnan(mixed[:, :M]).any()
    assert torch.equal(mixed[0, :M], companions[0, :M])
    assert torch.equal(mixed[1, :M], fp32[1, :M])


def test_live_row_count_decides_the_rows_written(geo):
    h, g, n, coords = geo["h"], geo["g"], geo["n"], geo["coords"]
    lvl, c1, cout = 1, 64, 96
    M = g.sizes()[lvl]
    og = ome.TensorField(torch.zeros(n, 1), coords).sparse().geom
    assert og.stride_level(2).shape[0] == M and og.stride_level(1).shape[0] == g.sizes()[0]
    W, A, _, R, sc_, sh_ = operands(27, c1, 0, cout, n, 11)
    Wp = h.pack_weights(W)
    nbr = g.nbr3[lvl]
    mask = g.mask_of[nbr.data_ptr()]
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    few = 128 * (sms // 2 - 10) + 3              # fewer live items (2 passes per tile) than SMs
    assert few < M
    ys = [ome.conv(ome.SparseTensor(A[p_][:M].double().cpu(), og, 2), W.double().cpu(), 3, 1, False).F for p_ in range(2)]
    for m in (1, 127, 129, few):
        d_m = torch.tensor([m], dtype=torch.int32, device=DEV)
        out = conv(h, W, Wp, A, None, R, sc_, sh_, nbr, n, d_m, mask=mask)
        for p_ in range(2):
            y = torch.relu(ys[p_][:m] * sc_.double().cpu() + sh_.double().cpu() + R[p_][:m].double().cpu())
            assert rel_err(out[p_][:m], y) < 5e-5, f"M = {m}, pass {p_}"
        assert torch.isnan(out[:, m:]).all(), f"M = {m}: a row beyond the live count was written"
