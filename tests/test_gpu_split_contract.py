"""Every producer of an fp16 hi/lo split writes the same bits: gate_mul's companions (all 2^32 fp32 inputs), the conv epilogues'
out_h / out_gated_h (tensor-core and FFMA kernels), and the A-operand image the tensor-core kernel splits from fp32 rows, which must
give the bits of the companion path.  Also decodes lb2_pack_weights' image: header, swizzled [hi | lo] tiles, zero channels, and the
power-of-two pre-scale at the edges of the float range.  The contract is restated in tests/split_numerics.py."""
import numpy as np
import pytest
import torch

import split_numerics as sn

pytestmark = pytest.mark.gpu
DEV, H, companion = sn.DEV, sn.handle, sn.companion


def test_gate_mul_companion_is_the_split_of_every_fp32():
    h = H()
    c, chunk = 1024, 1 << 26
    one = torch.ones(1, c, device=DEV)
    y = torch.empty(chunk // c, c, device=DEV)
    yh = torch.empty(chunk // c, 2 * c, dtype=torch.float16, device=DEV)
    for start in range(-(1 << 31), 1 << 31, chunk):
        x = torch.arange(start, start + chunk, dtype=torch.int64, device=DEV).to(torch.int32).view(torch.float32).view(-1, c)
        h.gate_mul(x, one, None, None, x.shape[0], c, y, yh)
        hi, lo = sn.split(x)
        assert sn.same_bits(y, x), f"x * 1 != x in [{start:#x}, +2^26)"
        assert sn.same_bits(yh[:, :c], hi) and sn.same_bits(yh[:, c:], lo), f"companion differs from the split in [{start:#x}, +2^26)"


@pytest.fixture(scope="module")
def geo():
    _, _, _, m_in, m_out, nbr = sn.case_map(27)
    return dict(m=m_out, nbr=nbr.to(DEV).contiguous(), d_m=torch.tensor([m_out], dtype=torch.int32, device=DEV))


def edge_tensor(shape, seed):
    """a tensor of `shape` whose entries are edge values, scaled powers of two and randn, in random positions"""
    g = torch.Generator().manual_seed(seed)
    e = sn.edge_values()
    n = int(np.prod(shape))
    pick = e[torch.randint(0, e.numel(), (n,), generator=g)]
    wide = torch.randn(n, generator=g) * 2.0 ** torch.randint(-30, 20, (n,), generator=g).float()
    return torch.where(torch.rand(n, generator=g) < 0.5, pick, wide).reshape(shape).contiguous()


@pytest.mark.parametrize("algo", [1, 2])
@pytest.mark.parametrize("kvol", [1, 27])
@pytest.mark.parametrize("cout", [32, 96, 256])
def test_epilogue_companions_are_the_split_of_the_fp32_outputs(geo, algo, kvol, cout):
    """W = 0, so y = residual (and y * gate) takes any chosen fp32 value; out_h / out_gated_h must be the split of the same
    launch's out / out_gated"""
    from lidiff_b200._lib import ConvDesc, ConvIO
    h = H()
    m, cin = geo["m"], 32
    W = torch.zeros(kvol, cin, cout, device=DEV)
    Wp = h.pack_weights(W)
    A = torch.randn(m, cin, device=DEV)
    R = edge_tensor((m, cout), cout + kvol).to(DEV)
    tab = torch.tensor([[1.0], [0.5], [3.0], [-2.0 ** 20]]).repeat(1, cout).to(DEV).contiguous()
    gi = torch.randint(0, 4, (m,), dtype=torch.int32, generator=torch.Generator().manual_seed(3)).to(DEV)
    out, outg = torch.empty(m, cout, device=DEV), torch.empty(m, cout, device=DEV)
    out_h, outg_h = (torch.empty(m, 2 * cout, dtype=torch.float16, device=DEV) for _ in range(2))
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = cin, 0, cout, kvol
    d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
    d.nbr = geo["nbr"].data_ptr() if kvol == 27 else None
    d.nbr_stride, d.d_mout, d.mout_cap, d.npass = m, geo["d_m"].data_ptr(), m, 1
    d.io[0] = ConvIO(A.data_ptr(), None, R.data_ptr(), out.data_ptr(), tab.data_ptr(), gi.data_ptr(), outg.data_ptr(), None,
                     None, None, out_h.data_ptr(), outg_h.data_ptr())
    h.spconv(d, algo)
    torch.cuda.synchronize()
    assert sn.same_bits(out, R + 0.0), "y = 0 + residual"
    for y, yh in ((out, out_h), (outg, outg_h)):
        hi, lo = sn.split(y)
        assert sn.same_bits(yh[:, :cout], hi) and sn.same_bits(yh[:, cout:], lo)
    assert torch.isinf(outg).any() and torch.isnan(outg_h).any() and torch.isinf(outg_h[:, cout:]).any()
    assert (outg_h[:, cout:].abs() == 65504).any(), "a value in (65504, 131024) whose low half is the largest fp16"


@pytest.fixture(scope="module")
def engine_geo():
    from lidiff_b200.engine import Geometry
    h = H()
    g = torch.Generator().manual_seed(47)
    pts = torch.randn(70_000, 3, generator=g) * 3.0
    coords = torch.cat([torch.zeros(70_000, 1), torch.round(pts / 0.05)], 1)
    G = Geometry(h, 70_000)
    G.build(coords.to(DEV).contiguous(), 70_000)
    return dict(h=h, g=G, n=70_000)


@pytest.mark.parametrize("c1,c2,cout,lvl", [(64, 32, 64, 2), (128, 0, 256, 3)])
def test_gather_paths_agree_at_the_edges(engine_geo, c1, c2, cout, lvl):
    """as test_passes_may_gather_by_different_paths, with activations from the edge set: pass 0 gathers the companions with
    cp.async, pass 1 splits the fp32 rows in registers; both passes see the same activations, so they give the same bits"""
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    h, G, n = engine_geo["h"], engine_geo["g"], engine_geo["n"]
    M = G.sizes()[lvl]
    nbr = G.nbr3[lvl]
    gen = torch.Generator().manual_seed(c1 + c2 + cout)
    W = (torch.randn(27, c1 + c2, cout, generator=gen) / np.sqrt((c1 + c2) * 27)).to(DEV)
    Wp = h.pack_weights(W)
    edge_rows = torch.rand(n, 1, generator=gen) < 0.03                  # rows of edge values among unit-scale rows, so that some
    A = torch.where(edge_rows, edge_tensor((n, c1), c1), torch.randn(n, c1, generator=gen)).to(DEV)   # outputs stay finite
    B = torch.where(edge_rows, edge_tensor((n, c2), c2 + 1), torch.randn(n, c2, generator=gen)).to(DEV) if c2 else None
    A_h, B_h = companion(h, A), (companion(h, B) if c2 else None)
    out = torch.full((2, n, cout), 7.0, device=DEV)
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, 27
    d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
    d.nbr, d.nbr_stride, d.d_mout, d.mout_cap, d.npass = nbr.data_ptr(), n, G.d_n[lvl].data_ptr(), n, 2
    d.row_perm, d.row_mask = G.perm3[lvl].data_ptr(), G.mask_of[nbr.data_ptr()].data_ptr()
    d.tile_order128 = G.tile_order_of[nbr.data_ptr()][0].data_ptr()
    for p_, use_h in ((0, True), (1, False)):
        d.io[p_] = ConvIO(A.data_ptr(), B.data_ptr() if c2 else None, None, out[p_].data_ptr(), None, None, None, None,
                          A_h.data_ptr() if use_h else None, B_h.data_ptr() if (use_h and c2) else None, None, None, None)
    h.spconv(d, _lib.ALGO_TC)
    torch.cuda.synchronize()
    assert sn.same_bits(out[0, :M], out[1, :M]), "the companion path and the fp32-row path disagree"
    fin = torch.isfinite(out[0, :M])
    assert fin.any() and (~fin).any()


# ---- packed weights ------------------------------------------------------------------------------------------------------
def decode_packed(P, kvol, cin, cout):
    """(header max|W| bits, header[1], hi (kvol, nchunks*64, cout) fp16, lo) of lb2_pack_weights' image"""
    P = P.cpu()
    nch = (cin + 63) // 64
    head = P[:8].view(torch.int32)
    tiles = P[256:].view(kvol, nch, 2, cout * 128)
    n = torch.arange(cout)[:, None]
    kk = torch.arange(64)[None, :]
    off = (n >> 3) * 1024 + (n & 7) * 128 + (((kk >> 3) ^ (n & 7)) << 4) + (kk & 7) * 2          # sw128(n, kk / 8) + 2 (kk % 8)
    idx = torch.stack([off, off + 1], -1)                                                           # the two bytes of a half
    img = tiles[:, :, :, idx].contiguous().view(torch.float16)[..., 0]                              # (kvol, nch, 2, cout, 64)
    hl = img.permute(2, 0, 1, 4, 3).reshape(2, kvol, nch * 64, cout)
    return int(head[0]), float(P[4:8].view(torch.float32)[0]), hl[0], hl[1]


@pytest.mark.parametrize("kvol,cin,cout", [(27, 48, 32), (8, 144, 96), (1, 64, 256)])
@pytest.mark.parametrize("mx", ["randn", "pow2", "below_pow2", "zero", "2^-120", "subnormal", "1e38", "FLT_MAX"])
def test_packed_weights_decode_to_the_split_of_w_times_2k(kvol, cin, cout, mx):
    h = H()
    g = torch.Generator().manual_seed(kvol * cin + cout)
    W = torch.randn(kvol, cin, cout, generator=g) / np.sqrt(cin * kvol)
    top = {"randn": None, "pow2": 0.125, "below_pow2": float(np.nextafter(np.float32(0.125), np.float32(0))), "zero": 0.0,
           "2^-120": 2.0 ** -120, "subnormal": 3e-42, "1e38": 1e38, "FLT_MAX": float(np.finfo(np.float32).max)}[mx]
    if top is not None:
        W = W / W.abs().max() * top if top > 0 else torch.zeros_like(W)
        W = W.float()
        if top > 0:
            W.view(-1)[5] = top                                     # the exact maximum
    W = W.float()
    P = h.pack_weights(W.to(DEV).contiguous())
    mbits, inv, hi, lo = decode_packed(P, kvol, cin, cout)
    m = np.float32(W.abs().max().item())
    assert mbits == int(np.array([m]).view(np.int32)[0])
    k = sn.weight_exponent(W)
    assert inv == 2.0 ** -k and np.isfinite(inv) and inv > 0
    assert inv >= 2.0 ** -126, "header[1] must be a normal fp32"
    if m > 0 and k < 126:
        assert 8192 <= float(m) * 2.0 ** k < 16384
    eh, el = sn.split(W * 2.0 ** k)
    assert sn.same_bits(hi[:, :cin], eh) and sn.same_bits(lo[:, :cin], el)
    assert (hi[:, cin:] == 0).all() and (lo[:, cin:] == 0).all(), "channels beyond cin must be zero"
    assert torch.isfinite(hi).all() and torch.isfinite(lo).all()
