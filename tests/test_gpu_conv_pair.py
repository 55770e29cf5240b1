"""Direct parity of the engine-path tensor-core convolution kernel against the fp64 oracle on its companion path (fp16 split
inputs `in1_h` / `in2_h` gathered with cp.async), with the engine's row order, row masks, two guidance passes, concatenated inputs
and the fused epilogue (BN affine + residual + ReLU + gate, fp32 and split outputs), for the Cout 128 and 256 layers of the
coarse levels.  Every case runs through both ways a caller reaches the kernel: LB2_ALGO_AUTO (0, the library's dispatch picks the
tensor-core variant for packed weights and a supported shape) and LB2_ALGO_TC (2, the tensor-core variant named directly)."""
import numpy as np
import pytest
import torch

from oracle import me_cpu as ome

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel_err(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs() / (b.abs() + b.pow(2).mean().sqrt() + 1e-30)).max().item()


@pytest.fixture(scope="module")
def geo():
    from lidiff_b200 import _lib
    from lidiff_b200.engine import Geometry
    h = _lib.get_handle(DEV)
    g = torch.Generator().manual_seed(77)
    n = 60_000
    pts = torch.randn(n, 3, generator=g) * torch.tensor([3.0, 3.0, 0.6])         # a slab: 10-20 neighbours per voxel on levels 2-4
    coords = torch.cat([torch.zeros(n, 1), torch.round(pts / 0.05)], 1)
    G = Geometry(h, n)
    G.build(coords.to(DEV).contiguous(), n)
    og = ome.TensorField(pts, coords).sparse().geom
    sizes = G.sizes()
    for l in range(5):
        assert sizes[l] == og.stride_level(1 << l).shape[0]
    return dict(h=h, G=G, og=og, n=n, sizes=sizes)


CASES = [  # c1, c2, cout, level of the output rows, map kind
    (256, 0, 256, 3, "3"), (256, 128, 256, 3, "3"), (384, 0, 256, 3, "1"), (256, 0, 256, 3, "up"), (128, 0, 256, 4, "3"),
    (128, 0, 128, 3, "3"), (128, 64, 128, 2, "3"), (256, 0, 128, 2, "up"), (64, 0, 128, 3, "3"), (128, 0, 128, 4, "dn"),
]


@pytest.mark.parametrize("algo", [0, 2])
@pytest.mark.parametrize("c1,c2,cout,lvl,kind", CASES)
def test_companion_path_kernels_match_fp64_oracle(geo, algo, c1, c2, cout, lvl, kind):
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    h, G, og, N = geo["h"], geo["G"], geo["og"], geo["n"]
    M = geo["sizes"][lvl]
    ts = 1 << lvl
    nbr, perm, kvol, lvl_in, oconv = {
        "3": (G.nbr3[lvl], G.perm3[lvl], 27, lvl, (ts, 3, 1, False)),
        "up": (G.nbr_up[lvl] if lvl < 4 else None, G.perm_up[lvl] if lvl < 4 else None, 8, lvl + 1, (2 * ts, 2, 2, True)),
        "dn": (G.nbr_dn[lvl] if lvl > 0 else None, G.perm_dn[lvl] if lvl > 0 else None, 8, lvl - 1, (ts // 2, 2, 2, False)),
        "1": (None, None, 1, lvl, (ts, 1, 1, False))}[kind]
    M_in = geo["sizes"][lvl_in]
    gen = torch.Generator().manual_seed(c1 * 7 + c2 + cout + lvl)
    W = torch.randn(kvol, c1 + c2, cout, generator=gen) / np.sqrt((c1 + c2) * kvol)
    A = torch.randn(2, N, c1, generator=gen)
    B = torch.randn(2, N, c2, generator=gen) if c2 else None
    R = torch.randn(2, N, cout, generator=gen)
    sc_, sh_ = torch.rand(cout, generator=gen) + 0.5, torch.randn(cout, generator=gen)
    tab = torch.randn(40, cout, generator=gen)
    gi = torch.randint(0, 40, (N,), generator=gen, dtype=torch.int32)
    d_ = lambda t: None if t is None else t.to(DEV).contiguous()
    dW, dA, dB, dR, dS, dT, dTab, dGi = map(d_, (W, A, B, R, sc_, sh_, tab, gi))
    Wp = h.pack_weights(dW)

    def split_of(x):                                   # fp16 hi/lo companion through the library's own split (gate_mul by 1)
        if x is None:
            return None
        c = x.shape[-1]
        one = torch.ones(1, c, device=DEV)
        xh = torch.zeros(2, N, 2 * c, dtype=torch.float16, device=DEV)
        for p_ in range(2):
            h.gate_mul(x[p_], one, None, None, N, c, torch.empty_like(x[p_]), xh[p_])
        return xh
    A_h, B_h = split_of(dA), split_of(dB)
    out, outg = torch.zeros(2, N, cout, device=DEV), torch.zeros(2, N, cout, device=DEV)
    out_h = torch.zeros(2, N, 2 * cout, dtype=torch.float16, device=DEV)
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, kvol
    d.weight, d.weight_packed = dW.data_ptr(), Wp.data_ptr()
    d.scale, d.shift, d.relu = dS.data_ptr(), dT.data_ptr(), 1
    d.nbr = nbr.data_ptr() if nbr is not None else None
    d.nbr_stride, d.d_mout, d.mout_cap, d.npass = N, G.d_n[lvl].data_ptr(), N, 2
    d.row_perm = perm.data_ptr() if perm is not None else None
    d.row_mask = G.mask_of[nbr.data_ptr()].data_ptr() if nbr is not None else None
    for p_ in range(2):
        d.io[p_] = ConvIO(dA[p_].data_ptr(), dB[p_].data_ptr() if dB is not None else None, dR[p_].data_ptr(), out[p_].data_ptr(),
                          dTab.data_ptr(), dGi.data_ptr() if p_ == 0 else None, outg[p_].data_ptr(), None,
                          A_h[p_].data_ptr(), B_h[p_].data_ptr() if B_h is not None else None, out_h[p_].data_ptr(), None)
    assert algo in (_lib.ALGO_AUTO, _lib.ALGO_TC)
    l0 = h.launch_count()
    h.spconv(d, algo)
    torch.cuda.synchronize()
    assert h.launch_count() - l0 == 1, "one conv launch (no split into a fallback path)"
    ts_in, ks, stride, tr = oconv
    for p_ in range(2):
        Fin = A[p_][:M_in] if B is None else torch.cat([A[p_][:M_in], B[p_][:M_in]], 1)
        y = ome.conv(ome.SparseTensor(Fin.double(), og, ts_in), W.double(), ks, stride, tr).F
        assert y.shape[0] == M
        y = torch.relu(y * sc_.double() + sh_.double() + R[p_][:M].double())
        e = rel_err(out[p_][:M], y)
        gate = tab[gi[:M].long()] if p_ == 0 else tab[0:1]
        eg = rel_err(outg[p_][:M], y * gate.double())
        oh = out_h[p_][:M].float().cpu()
        es = rel_err(oh[:, :cout] + oh[:, cout:], y)
        print(f"algo={algo} {c1}+{c2}->{cout} L{lvl} {kind} pass {p_}: rel err {e:.2e} gated {eg:.2e} split {es:.2e}")
        assert e < 5e-5 and eg < 5e-5 and es < 5e-5, "tensor-core conv (companion path) vs fp64 oracle"
    assert out[:, M:].abs().sum() == 0, "rows beyond the live count must stay untouched"
