"""TEST INFRASTRUCTURE: the fp16 hi/lo split of the tensor-core convolutions restated on the host, the numerics cases shared by
tests/test_gpu_conv_numerics.py (the kernels) and tests/test_split_numerics_host.py (host emulations), and the error model both
hold them to.

Split contract (tc::split2 in lidiff_b200/csrc/tc_common.cuh), RN = round to nearest-even to fp16 (overflow to +-inf), RN_sat =
RN with a result beyond the fp16 range, infinities included, clamped to +-65504 (NaN stays NaN):
    hi = RN_sat(x),  lo = RN(fp32(x - hi))
so for |x| < 131024 hi + lo = x to 2^-22, and for larger |x|, +-inf included, lo = +-inf; NaN gives hi = lo = NaN.  A value the
split cannot hold therefore makes every product that reads it non-finite.

Error model of one output y = sum_i x_i w_i of the FP16x3 convolution (weights pre-scaled by s = 2^k, max|W| s in [8192, 16384)):
  * Representation.  For |x| <= 65504, x - hi is exact in fp32 and |x - hi| <= 2^-11 |x|; rounding it to fp16 costs 2^-11 of it
    while it is a normal fp16, and at most half the subnormal spacing, 2^-25, below 2^-14.  So |x - hi - lo| <= 2^-22 |x| + 2^-25
    (the low half is subnormal below |x| = 2^-3, and |x| < 2^-25 splits to zero).  The same holds for w s.  The kernel forms
    x_hi w_hi + x_lo w_hi + x_hi w_lo; the dropped x_lo w_lo is <= 2^-22 |x w s| (plus terms of order 2^-35 |x w s|).  Per
    product that is <= (3 + 2^-9) 2^-22 |x w s| + (1 + 2^-20) 2^-25 (|w s| + |x|); unscaled by s and summed:
        REP = 3.002 * 2^-22 * S1 + 1.001 * 2^-25 * (sum|w| + 2^-k sum|x|),   S1 = sum |x_i w_i|.
  * Accumulation.  The rounding inside wgmma is not documented.  Model it as at most one fp32 ulp of the partial sum, <= 2^-23 S1,
    per MMA instruction of an accumulation chain.  A chain holds 3 ceil(c_tot / 16) instructions per kernel offset for `group`
    offsets (group = max(1, 64 // (3 ceil(c_tot / 16))), as the kernel cuts them); after each group one round-to-nearest add
    (<= 2^-24 S1) into the running total.  ACC = (n_chain 2^-23 + n_groups 2^-24) S1.
    The scatter split (lb2_spconv_scatter + the centre offset as a 1x1 convolution with pre_add) accumulates differently: one chain
    of 3 ceil(c_tot / 16) instructions per kernel offset (each <= 2^-23 of its own offset's S1, together <= n_chain 2^-23 S1 with
    n_chain = 3 ceil(c_tot / 16)), then up to kvol - 1 fp32 atomic adds into the pre_add buffer and the epilogue's add of pre_add,
    each one RN add: n_groups = kvol.  Same formulas, with these counts (chain(ctot, kvol, "scatter")).
  * Hard bound, every element:   |y - y64| <= tau_h S1 + 1.001 * 2^-25 (sum|w| + 2^-k sum|x|),
        tau_h = 3.002 * 2^-22 + n_chain 2^-23 + n_groups 2^-24.
  * Statistical bound, per case.  With the floors folded into the magnitudes (|x~| = max(|x|, 2^-3), |w~| = max(|w|, 2^-3-k), so
    that |x - hi - lo| <= 2 * 2^-22 |x~|), one product's representation error is <= 5 * 2^-22 |x~ w~|.  Taken as independent and
    uniform, their sum has sigma <= 5 * 2^-22 / sqrt(3) * sqrt(S2~), S2~ = sum x~^2 w~^2.  A partial sum of random-sign products
    stays below Z sqrt(S2~), so the accumulation adds at most Z (n_chain 2^-23 + n_groups 2^-24) sqrt(S2~).  With Z = 6 (a 6-sigma
    excursion; no case has more than 10^7 outputs):
        max |y - y64| / sqrt(S2~) <= tau_s = Z (5 * 2^-22 / sqrt(3) + n_chain 2^-23 + n_groups 2^-24).
    The accumulation term is summed linearly, not as sqrt(n_chain): how wgmma aligns and rounds its partial sums is not documented,
    and alignment by truncation rounds toward zero, an error of the same sign at every instruction of a chain.  Errors that may all
    point one way cannot be assumed to cancel, so tau_s (about 5e-5 at most shapes) is a bound, not an estimate: the measured
    FP16x3 error sits far below it, and a defect of the accumulation that stays within this linear budget passes unnoticed.
    A dropped cross term x_lo w_hi is a random-sign error of about 2^-12 / sqrt(3) |x w| per product, ~50x the representation sigma:
    the statistical bound rejects it (tests/test_split_numerics_host.py), the hard bound alone would not.
  * The FFMA kernel (fp32 operands, one fma per product in a chain of N = c_tot * kvol products): each fma rounds once,
    <= 2^-24 of the partial sum.  Hard: |y - y64| <= N 2^-24 S1.  Statistical: Z sqrt(N) 2^-24 Z sqrt(S2) (RN errors of random sign
    on partial sums below Z sqrt(S2)).
"""
import math

import numpy as np
import torch

from oracle import me_cpu as ome

FP16_MAX = 65504.0
Z = 6.0


# ---- the split contract --------------------------------------------------------------------------------------------------
def rn_sat(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> fp16, round to nearest-even, values beyond the fp16 range (infinities included) clamped to +-65504 (a plain fp16
    cast overflows to inf instead), NaN kept NaN"""
    h = x.to(torch.float16)
    return torch.where(torch.isinf(h), torch.copysign(torch.full_like(h, FP16_MAX), h), h)


def split(x: torch.Tensor):
    """(hi, lo) fp16 of fp32 x under the split contract"""
    x = x.float()
    hi = rn_sat(x)
    return hi, (x - hi.float()).to(torch.float16)


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """equal bit for bit, except that any NaN matches any NaN"""
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    ia = a.view(torch.int16 if a.dtype == torch.float16 else torch.int32)
    ib = b.view(torch.int16 if b.dtype == torch.float16 else torch.int32)
    return bool(((ia == ib) | na).all())


def edge_values() -> torch.Tensor:
    """fp32 values where a split goes wrong: subnormals, +-0, 2^-25 .. 2^-3, 65504 +- ulp, 131008 +- ulp, FLT_MAX, +-inf, NaN"""
    f = np.float32
    v = [0.0, -0.0, 1e-45, -1e-45, 1e-40, 2.0 ** -126, -(2.0 ** -126) * 1.5, 1.0, -1.0, 3.0, 2.0 ** -24, 2.0 ** -14]
    for e in range(-25, -2):
        v += [2.0 ** e, -(2.0 ** e) * 1.3, 2.0 ** e * 1.0009765625]
    for c in (65504.0, 65520.0, 131008.0, 2.0 ** 16, 2.0 ** 17):
        v += [c, -c, float(np.nextafter(f(c), f(np.inf))), float(np.nextafter(f(c), f(0)))]
    v += [float(np.finfo(np.float32).max), -float(np.finfo(np.float32).max), 1e30, -3e20, 40000.7, -65519.99]
    v += [math.inf, -math.inf, math.nan]
    return torch.tensor(v, dtype=torch.float32)


# ---- GPU helpers shared by the GPU test files (the library is imported only when they run) ----------------------------------------
DEV = "cuda:0"


def handle():
    from lidiff_b200 import _lib
    return _lib.get_handle(DEV)


def companion(h, x):
    """fp16 split companion (n, 2c) of a device tensor x (n, c), written by lb2_gate_mul with a gate of ones"""
    n, c = x.shape
    y, yh = torch.empty_like(x), torch.empty(n, 2 * c, dtype=torch.float16, device=DEV)
    h.gate_mul(x, torch.ones(1, c, device=DEV), None, None, n, c, y, yh)
    return yh


# ---- weight pre-scale of lb2_pack_weights ------------------------------------------------------------------------------------
def weight_exponent(w: torch.Tensor) -> int:
    """k of the packer: max|W| 2^k in [8192, 16384), capped at 126 so that 2^k and 2^-k stay finite, nonzero and normal; 0 for
    all-zero W"""
    m = np.float32(w.abs().max().item())
    if not (m > 0) or not np.isfinite(m):
        return 0
    _, e = np.frexp(m)
    return min(14 - int(e), 126)


# ---- numerics cases ----------------------------------------------------------------------------------------------------------
# c1, c2, cout, kvol, p (activations ~ 2^p randn, |randn| <= 1.99), outlier (one weight 2^12 above the rest)
CASES = [
    (16, 0, 32, 27, 0, False), (48, 0, 64, 27, 0, False), (80, 0, 96, 8, 0, False), (144, 0, 128, 27, 0, False),
    (384, 0, 256, 27, 0, False),                                 # long K: group = 1, a chain is 72 MMAs (> STEP_BUDGET)
    (16, 16, 32, 27, 0, False), (48, 32, 64, 27, 0, False), (80, 64, 128, 8, 0, False), (128, 64, 128, 1, 0, False),
    (64, 0, 64, 27, -24, False), (64, 0, 64, 27, -12, False), (64, 0, 64, 27, -4, False), (64, 0, 64, 27, 8, False),
    (64, 0, 64, 27, 15, False), (96, 0, 96, 27, 0, True), (48, 0, 256, 1, 0, False),
]


def case_id(c):
    c1, c2, cout, kvol, p, outlier = c
    return f"{c1}+{c2}to{cout}_k{kvol}_p{p}" + ("_outlier" if outlier else "")


_FIELD = {}


def field():
    """one point cloud (~13 k level-0 voxels, ~8 neighbours each) with its oracle geometry"""
    if not _FIELD:
        g = torch.Generator().manual_seed(2024)
        pts = torch.randn(40_000, 3, generator=g) * torch.tensor([0.5, 0.5, 0.12])
        coords = torch.cat([torch.zeros(pts.shape[0], 1), torch.round(pts / 0.05)], 1)
        _FIELD["geom"] = ome.TensorField(pts, coords).sparse().geom
    return _FIELD["geom"]


def case_map(kvol):
    """(ts_in, ks, stride, m_in, m_out, nbr (kvol, m_out) int32 with -1 = no neighbour, or None for the 1x1 identity)"""
    og = field()
    if kvol == 1:
        m = og.stride_level(1).shape[0]
        return 1, 1, 1, m, m, None
    ks, stride = (3, 1) if kvol == 27 else (2, 2)
    maps = og.kernel_map(1, ks, stride, False)
    m_in, m_out = og.stride_level(1).shape[0], og.stride_level(stride).shape[0]
    nbr = torch.full((kvol, m_out), -1, dtype=torch.int32)
    for k, (i_rows, o_rows) in enumerate(maps):
        nbr[k, torch.from_numpy(o_rows)] = torch.from_numpy(i_rows).int()
    return 1, ks, stride, m_in, m_out, nbr


def case_operands(c):
    """(X (m_in, c_tot) fp32, W (kvol, c_tot, cout) fp32) of a case, seeded by its shape"""
    c1, c2, cout, kvol, p, outlier = c
    ctot = c1 + c2
    _, _, _, m_in, _, _ = case_map(kvol)
    g = torch.Generator().manual_seed(ctot * 1009 + cout * 31 + kvol + 7 * (p + 30) + outlier)
    X = (torch.randn(m_in, ctot, generator=g).clamp(-1.99, 1.99) * 2.0 ** p).float()
    W = (torch.randn(kvol, ctot, cout, generator=g) / math.sqrt(ctot * kvol)).float()
    if outlier:
        W[kvol // 2, ctot // 3, cout // 5] = W.abs().max() * 4096.0
    return X, W


def conv64(kvol, X, W):
    """oracle.me_cpu.conv in fp64 on the case's map"""
    ts, ks, stride, _, _, _ = case_map(kvol)
    W = W.double()
    return ome.conv(ome.SparseTensor(X.double(), field(), ts), W[0] if kvol == 1 else W, ks, stride, False).F


def chain(ctot, kvol, path="tc"):
    """(MMA instructions in the longest accumulation chain, RN adds of partial sums per output) of k_spconv_tc, or of the
    scatter split (path "scatter")"""
    steps = 3 * ((ctot + 15) // 16)
    if path == "scatter":
        return steps, kvol
    group = max(1, 64 // steps)
    return steps * min(group, kvol), (kvol + group - 1) // group


def tau_h(ctot, kvol, path="tc"):
    n, g = chain(ctot, kvol, path)
    return 3.002 * 2.0 ** -22 + n * 2.0 ** -23 + g * 2.0 ** -24


def tau_s(ctot, kvol, path="tc"):
    n, g = chain(ctot, kvol, path)
    return Z * (5 * 2.0 ** -22 / math.sqrt(3) + n * 2.0 ** -23 + g * 2.0 ** -24)


def tau_ffma(ctot, kvol):
    """(hard, statistical) bars of the fp32 FFMA kernel"""
    n = ctot * kvol
    return n * 2.0 ** -24, Z * Z * math.sqrt(n) * 2.0 ** -24


class Reference:
    """fp64 output of a case and the per-element scales of the error model"""

    def __init__(self, c, X=None, W=None, k=None):
        c1, c2, cout, kvol, p, outlier = c
        if X is None:
            X, W = case_operands(c)
        self.ctot, self.kvol = c1 + c2, kvol
        self.k = weight_exponent(W) if k is None else k          # k of the packed weights (W may be a part of them)
        Xa, Wa = X.double().abs(), W.double().abs()
        self.y = conv64(kvol, X, W)
        self.S1 = conv64(kvol, Xa, Wa)
        self.S2 = conv64(kvol, Xa ** 2, Wa ** 2)
        Xf, Wf = Xa.clamp(min=2.0 ** -3), Wa.clamp(min=2.0 ** (-3 - self.k))
        self.S2f = conv64(kvol, Xf ** 2, Wf ** 2)
        sw = conv64(kvol, torch.ones_like(Xa), Wa)
        sx = conv64(kvol, Xa, torch.ones(kvol, self.ctot, 1, dtype=torch.float64))
        self.floor = 1.001 * 2.0 ** -25 * (sw + 2.0 ** -self.k * sx)

    def errors(self, y, ffma=False, path="tc"):
        """(hard-bound ratio: max err / bound, <= 1 passes; statistical: max err / sqrt(S2~) (S2 for the fp32 model))"""
        err = (y.double().cpu() - self.y).abs()
        if ffma:
            th, _ = tau_ffma(self.ctot, self.kvol)
            return (err / (th * self.S1 + 1e-300)).max().item(), (err / self.S2.sqrt().clamp(min=1e-300)).max().item()
        bound = tau_h(self.ctot, self.kvol, path) * self.S1 + self.floor
        return (err / bound).max().item(), (err / self.S2f.sqrt()).max().item()


# ---- host emulation of the kernel's products -----------------------------------------------------------------------------------
def emulate(c, X, W, scheme="f16x3"):
    """the convolution as FP16x3 forms it: restated split of X and of W 2^k, the three products summed in fp32 (RN), times 2^-k.
    scheme "f16x2": no x_lo w_hi term; "f16x3_last": both cross terms dropped in the channels of a last partial 64-channel chunk."""
    c1, c2, cout, kvol, p, outlier = c
    ctot = c1 + c2
    k = weight_exponent(W)
    xh, xl = (t.float() for t in split(X))
    wh, wl = (t.float() for t in split(W * 2.0 ** k))
    if scheme == "f16x2":
        xl = torch.zeros_like(xl)
    elif scheme == "f16x3_last":
        last = (ctot // 64) * 64
        xl, wl = xl.clone(), wl.clone()
        xl[:, last:] = 0
        wl[:, last:, :] = 0
    elif scheme != "f16x3":
        raise ValueError(scheme)
    ts, ks, stride, _, m_out, nbr = case_map(kvol)
    out = torch.zeros(m_out, cout, dtype=torch.float32)
    maps = [(np.arange(m_out), np.arange(m_out))] if kvol == 1 else field().kernel_map(ts, ks, stride, False)
    for kk, (i_rows, o_rows) in enumerate(maps):
        if i_rows.shape[0]:
            i_t, o_t = torch.from_numpy(i_rows), torch.from_numpy(o_rows)
            a_h, a_l = xh[i_t], xl[i_t]
            part = a_h @ wh[kk] + a_l @ wh[kk] + a_h @ wl[kk]
            out.index_add_(0, o_t, part)
    return out * 2.0 ** -k
