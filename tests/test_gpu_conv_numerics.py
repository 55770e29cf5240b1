"""Element-wise accuracy of the sparse convolutions against oracle.me_cpu.conv in fp64, at the shapes, scales and values where an
FP16x3 split loses bits.  Every output element gets its own scale from the same map: S1 = conv(|X|, |W|), S2 = conv(X^2, W^2),
sum|w| = conv(1, |W|), sum|x| = conv(|X|, 1).  The bars come from the error model written out in tests/split_numerics.py:
  * hard, every element:  |y - y64| <= tau_h S1 + 2^-25 (sum|w| + 2^-k sum|x|), tau_h from the chain lengths the kernel runs;
  * statistical, per case:  max |y - y64| / sqrt(S2~) <= tau_s, S2~ = S2 with |x| and |w 2^k| floored at 2^-3 (below it the split
    has an absolute error floor of 2^-25);
  * the FFMA kernel under the fp32 model (one rounding per fma).
tests/test_split_numerics_host.py shows on the host that tau_s rejects FP16x2 and a dropped cross term in the last partial chunk.
Each case prints both normalised errors next to its bars."""
import numpy as np
import pytest
import torch

import split_numerics as sn

pytestmark = pytest.mark.gpu
DEV, H, companion = sn.DEV, sn.handle, sn.companion


def run_conv(h, c, X, W, algo, use_h=False, scale=None, shift=None):
    """one launch of lb2_spconv_forward on the case's map; X (m_in, c1 + c2) and W on the host"""
    from lidiff_b200._lib import ConvDesc, ConvIO
    c1, c2, cout, kvol = c[:4]
    _, _, _, m_in, m_out, nbr = sn.case_map(kvol)
    dX, dW = X.to(DEV), W.to(DEV).contiguous()
    A, B = dX[:, :c1].contiguous(), (dX[:, c1:].contiguous() if c2 else None)
    A_h, B_h = (companion(h, A), companion(h, B) if c2 else None) if use_h else (None, None)
    Wp = h.pack_weights(dW) if algo != 1 else None
    nb = nbr.to(DEV).contiguous() if nbr is not None else None
    d_m = torch.tensor([m_out], dtype=torch.int32, device=DEV)
    out = torch.full((m_out, cout), float("nan"), device=DEV)
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, kvol
    d.weight, d.weight_packed = dW.data_ptr(), (Wp.data_ptr() if Wp is not None else None)
    if scale is not None:
        ds, dt = scale.to(DEV).contiguous(), shift.to(DEV).contiguous()
        d.scale, d.shift = ds.data_ptr(), dt.data_ptr()
    d.nbr = nb.data_ptr() if nb is not None else None
    d.nbr_stride, d.d_mout, d.mout_cap, d.npass = m_out, d_m.data_ptr(), m_out, 1
    d.io[0] = ConvIO(A.data_ptr(), B.data_ptr() if c2 else None, None, out.data_ptr(), None, None, None, None,
                     A_h.data_ptr() if A_h is not None else None, B_h.data_ptr() if B_h is not None else None, None, None, None)
    h.spconv(d, algo)
    torch.cuda.synchronize()
    return out.cpu()


def run_scatter(h, c, X, W, use_h=False, centre=True):
    """the gather-GEMM-scatter split of a 3^3 convolution: off-centre pairs scattered into `pre`, then the centre 1x1 with pre_add
    (centre=False: `pre` itself, the sum over the 26 off-centre offsets)"""
    from lidiff_b200._lib import ConvDesc, ConvIO, ScatterDesc
    c1, c2, cout, kvol = c[:4]
    _, _, _, m_in, m, nbr = sn.case_map(kvol)
    nb = nbr.to(DEV).contiguous()
    d_m = torch.tensor([m], dtype=torch.int32, device=DEV)
    i32 = dict(dtype=torch.int32, device=DEV)
    pin, pout = torch.zeros(26 * m, **i32), torch.zeros(26 * m, **i32)
    koff, toff, scr = torch.zeros(28, **i32), torch.zeros(28, **i32), torch.zeros(64, **i32)
    h.pair_list(nb, m, d_m, m, 27, 13, pin, pout, koff, toff, scr)
    dX, dW = X.to(DEV), W.to(DEV).contiguous()
    A, B = dX[:, :c1].contiguous(), (dX[:, c1:].contiguous() if c2 else None)
    Wp, Wc = h.pack_weights(dW), dW[13:14].contiguous()
    Wpc = h.pack_weights(Wc)
    pre = torch.full((m, cout), 7.0, device=DEV)
    sd = ScatterDesc()
    sd.c1, sd.c2, sd.cout, sd.kvol, sd.npass = c1, c2, cout, 27, 1
    sd.weight_packed, sd.pair_in, sd.pair_out, sd.koff, sd.tile_off = Wp.data_ptr(), pin.data_ptr(), pout.data_ptr(), koff.data_ptr(), toff.data_ptr()
    sd.in1[0], sd.in2[0], sd.out[0] = A.data_ptr(), (B.data_ptr() if c2 else None), pre.data_ptr()
    if use_h:
        A_h, B_h = companion(h, A), (companion(h, B) if c2 else None)
        sd.in1_h[0], sd.in2_h[0] = A_h.data_ptr(), (B_h.data_ptr() if c2 else None)
    sd.d_zero_rows, sd.zero_rows_cap = d_m.data_ptr(), m
    h.spconv_scatter(sd)
    if not centre:
        torch.cuda.synchronize()
        return pre.cpu()
    out = torch.full((m, cout), float("nan"), device=DEV)
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, 1
    d.weight, d.weight_packed = Wc.data_ptr(), Wpc.data_ptr()
    d.d_mout, d.mout_cap, d.npass = d_m.data_ptr(), m, 1
    d.io[0] = ConvIO(A.data_ptr(), B.data_ptr() if c2 else None, None, out.data_ptr(), None, None, None, pre.data_ptr())
    h.spconv(d, 2)
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("c", sn.CASES, ids=sn.case_id)
def test_tensor_core_conv_inside_the_error_model(c):
    h = H()
    X, W = sn.case_operands(c)
    ref = sn.Reference(c, X, W)
    paths = {"fp32": run_conv(h, c, X, W, 2), "companion": run_conv(h, c, X, W, 2, use_h=True)}
    c1, c2, cout, kvol = c[:4]
    if kvol == 27 and h.scatter_supported(c1, c2, cout, 27):
        paths["scatter"] = run_scatter(h, c, X, W)
    for name, y in paths.items():
        path = "scatter" if name == "scatter" else "tc"
        th, ts = sn.tau_h(ref.ctot, ref.kvol, path), sn.tau_s(ref.ctot, ref.kvol, path)
        eh, es = ref.errors(y, path=path)
        print(f"NUMERICS {sn.case_id(c)} {name}: hard {eh:.3f} of bound (tau_h {th:.2e}), stat {es:.2e} (tau_s {ts:.2e})")
        assert eh <= 1.0, name
        assert es <= ts, name


@pytest.mark.parametrize("use_h", [False, True])
@pytest.mark.parametrize("c", [(8, 8, 32, 27, 0, False), (40, 24, 64, 27, 0, False), (72, 56, 128, 27, 0, False)], ids=sn.case_id)
def test_scatter_concat_boundary_inside_a_k_step(c, use_h):
    """lb2_spconv_scatter takes concatenated inputs with c1 % 8 == 0 (lb2_spconv_forward needs c1 % 16 == 0 when in2 is given), so
    the c1 | c2 boundary can fall inside a 16-channel k-step: its sum over the 26 off-centre offsets against fp64"""
    X, W = sn.case_operands(c)
    Wz = W.clone()
    Wz[13] = 0                                                      # the centre offset is not the scatter kernel's
    ref = sn.Reference(c, X, Wz, k=sn.weight_exponent(W))
    h = H()
    assert h.scatter_supported(c[0], c[1], c[2], 27)
    eh, es = ref.errors(run_scatter(h, c, X, W, use_h, centre=False), path="scatter")
    ts = sn.tau_s(ref.ctot, 27, "scatter")
    print(f"NUMERICS {sn.case_id(c)} scatter-only{' companion' if use_h else ''}: hard {eh:.3f} of bound, stat {es:.2e} (tau_s {ts:.2e})")
    assert eh <= 1.0 and es <= ts


FFMA_CASES = [(3, 0, 32, 27, 0, False), (20, 0, 7, 27, 0, False), (64, 0, 64, 27, -12, False), (48, 0, 64, 27, 0, False),
              (80, 0, 96, 8, 0, False)]


@pytest.mark.parametrize("c", FFMA_CASES, ids=sn.case_id)
def test_ffma_conv_inside_the_fp32_model(c):
    X, W = sn.case_operands(c)
    ref = sn.Reference(c, X, W)
    eh, es = ref.errors(run_conv(H(), c, X, W, 1), ffma=True)
    th, ts = sn.tau_ffma(ref.ctot, ref.kvol)
    print(f"NUMERICS {sn.case_id(c)} ffma: hard {eh:.3f} of bound (N 2^-24 = {th:.2e}), stat {es:.2e} (bar {ts:.2e})")
    assert eh <= 1.0 and es <= ts


@pytest.mark.parametrize("c", [(64, 0, 64, 27, 0, False), (80, 64, 128, 8, 0, False), (48, 0, 256, 1, 0, False)], ids=sn.case_id)
def test_per_output_channel_scales_undone_by_bn(c):
    """weights of output channel n scaled by 2^e_n, e_n in -10 .. 10, and BN scale 2^-e_n: the layer-wide pre-scale follows the
    largest channel, so the small ones lose bits to the 2^-25 floor.  Every channel's error after the epilogue must stay inside its
    own bound; the global |a - b| / (|b| + rms(b)) metric cannot see an error confined to one channel."""
    cout = c[2]
    X, W = sn.case_operands(c)
    e = torch.linspace(-10, 10, cout).round()
    Ws = (W * 2.0 ** e).float()
    ref = sn.Reference(c, X, Ws)
    scale, shift = (2.0 ** -e).float(), torch.zeros(cout)
    y = run_conv(H(), c, X, Ws, 2, scale=scale, shift=shift).double()
    y64 = ref.y * scale.double()
    bound = (sn.tau_h(ref.ctot, ref.kvol) * ref.S1 + ref.floor) * scale.double() + 2.0 ** -24 * y64.abs()
    ratio = ((y - y64).abs() / bound).amax(0)
    rel = ((y - y64).abs().amax(0) / y64.abs().amax(0))
    print(f"NUMERICS {sn.case_id(c)} per-channel: worst channel {ratio.max():.3f} of its bound; rel err 2^-10 channel "
          f"{rel[0]:.2e}, 2^0 {rel[cout // 2]:.2e}, 2^10 {rel[-1]:.2e}")
    assert (ratio <= 1.0).all(), f"channels over their bound: {torch.nonzero(ratio > 1).flatten().tolist()}"


@pytest.mark.parametrize("algo,use_h", [(2, False), (2, True), (1, False)])
@pytest.mark.parametrize("c", [(64, 0, 64, 27, 0, False), (128, 64, 256, 27, 0, False)], ids=sn.case_id)
def test_non_finite_rows_reach_exactly_their_outputs(c, algo, use_h):
    """a NaN row and a +-inf row of the input: the set of non-finite outputs is the fp64 reference's, through either gather path of
    the tensor-core kernel and through the FFMA kernel, and every other output has the bits of a run with those rows zeroed (MMA
    rows are independent)."""
    h = H()
    X, W = sn.case_operands(c)
    X0 = X.clone()
    r_nan, r_inf = 17, X.shape[0] // 2
    X0[[r_nan, r_inf]] = 0
    Xb = X0.clone()
    Xb[r_nan] = float("nan")
    Xb[r_inf] = torch.where(torch.arange(X.shape[1]) % 2 == 0, torch.tensor(float("inf")), torch.tensor(-float("inf")))
    y64 = sn.conv64(c[3], Xb, W)
    y, y0 = run_conv(h, c, Xb, W, algo, use_h), run_conv(h, c, X0, W, algo, use_h)
    bad = ~torch.isfinite(y64)
    assert bad.any()
    assert torch.equal(~torch.isfinite(y), bad), "non-finite outputs differ from the fp64 reference's"
    assert sn.same_bits(y[~bad], y0[~bad]), "a row that does not read the non-finite rows changed"


@pytest.mark.parametrize("use_h", [False, True])
@pytest.mark.parametrize("value", [float("inf"), float("nan")])
@pytest.mark.parametrize("c", [(64, 0, 64, 27, 0, False), (128, 64, 256, 27, 0, False)], ids=sn.case_id)
def test_non_finite_weight_reaches_only_its_output_channel(c, value, use_h):
    """one +inf or NaN weight W[k][i][j]: the packer's pre-scale follows the largest finite weight, so every output outside channel
    j has the bits of a run with that weight zeroed, and channel j is non-finite wherever the fp64 reference is.  An output row
    without neighbour k multiplies the weight by a zero-filled row (0 * inf = NaN), so channel j may be non-finite there too."""
    h = H()
    X, W = sn.case_operands(c)
    k, i, j = 5, 7, c[2] // 3
    W0 = W.clone()
    W0[k, i, j] = 0
    Wb = W0.clone()
    Wb[k, i, j] = value
    y, y0 = run_conv(h, c, X, Wb, 2, use_h), run_conv(h, c, X, W0, 2, use_h)
    ref_bad, bad = ~torch.isfinite(sn.conv64(c[3], X, Wb)), ~torch.isfinite(y)
    assert ref_bad.any()
    assert bad[ref_bad].all(), "an output that reads the non-finite weight is finite"
    others = torch.ones_like(bad)
    others[:, j] = False
    assert not bad[others].any(), "a non-finite output outside the weight's channel"
    assert sn.same_bits(y[others], y0[others]), "an output of another channel changed"
