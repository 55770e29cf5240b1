"""TEST INFRASTRUCTURE: the error model of the sparse convolution's gradients, shared by tests/test_gpu_grad_numerics.py (the
kernels) and tests/test_grad_numerics_host.py (host emulations of the weight gradient's products).  Nothing here imports the CUDA
library; every helper runs on whatever device its tensors live on.

Weight gradient, lb2_spconv_wgrad (csrc/spconv_wgrad.cu):  dW[k] (cin x cout) = sum over output rows o with nbr[k][o] >= 0 of
X[nbr[k][o]]^T G[o], a reduction over the output rows.
  * Operands.  X is split like an activation (tc::split2, tests/split_numerics.py): no scale, |x - hi - lo| <= 2^-22 |x| + 2^-25, and
    non-finite from |x| >= 131024 on.  G is split like a weight after the pre-scale s = 2^k, max|G| s in [8192, 16384) over the
    finite elements of G, k capped at 126.  Per product the representation error is that of the forward model, unscaled by s:
        REP <= 3.002 * 2^-22 |x g| + 1.001 * 2^-25 (|g| + 2^-k |x|).
    That takes |x_lo| <= 2^-11 |x|, which fails for 65504 < |x| < 131024: hi saturates at 65504 and lo holds the rest, so the
    dropped x_lo (g s)_lo adds up to 1.001 (|x| - 65504) (2^-11 |g| + 2^-25 2^-k) per product.  The hard bar adds this saturation
    allowance (zero for every other x) and the statistical bar is taken over the error beyond it.  The forward model has the same
    term for saturated activations; its cases stay below 65504.
  * Chains.  A CTA cuts its chunk of rows into stages of BR = 64 rows; a stage with no neighbour issues no MMAs.  A chain is one
    group of at most GROUP = 5 live stages x 4 k-steps x 3 MMAs = 60 wgmma instructions (empty stages do not count toward a
    group), each modelled as at most one fp32 ulp of the partial sum, <= 2^-23 S1.
  * Adds.  One RN fold of each group into the chunk's fp32 total, at most ceil(rows_per_chunk / 320) per chunk, then nchunks - 1 RN
    adds of the chunk partials in k_wgrad_reduce, each <= 2^-24 S1.  The final x 2^-k is exact unless the result is an fp32
    subnormal, where it rounds once: <= 2^-150 absolute.
  * Hard bound, every element:  |dW - dW64| <= tau_h S1 + 1.001 * 2^-25 (sum|g| + 2^-k sum|x|) + 2^-150,
        tau_h = 3.002 * 2^-22 + n_chain 2^-23 + n_adds 2^-24.
  * Statistical bound, per case:  max |dW - dW64| / sqrt(S2~) <= tau_s = Z (5 * 2^-22 / sqrt(3) + n_chain 2^-23 + n_adds 2^-24),
    S2~ = sum x~^2 g~^2 with |x~| = max(|x|, 2^-3), |g~| = max(|g|, 2^(-3-k)), Z = 6: the reasoning of split_numerics.py.
    Here the reduction runs over up to ~10^6 rows per element: tau_h S1 grows with the row count N, a random-sign error of a
    dropped term only with sqrt(N), so only the statistical bar sees a dropped cross term at scan-sized N.
  * Non-finite values.  A NaN or +-inf in X (or |x| >= 131024) makes exactly the dW elements that read it non-finite; a NaN or +-inf
    in G likewise.  They do not enter the pre-scale, so every other element has the bits of a run with them zeroed.

Input gradient (me._ConvBase._input_grad): the forward kernel on the adjoint map, activation operand G s (s = 2^e from the largest
finite |G|, max|G s| in [8192, 16384), e capped at 126), weight operand the transformed kernel W_adj^T, packed per output slice with
its own 2^k.  The forward model of split_numerics.py applied to (G s, W_adj^T) and unscaled by s: hard bound tau_h S1 +
1.001 * 2^-25 (sum|w| / s + 2^-k sum|g|) + 2^-150 (the final / s rounds only into the subnormals); statistical bound with
|g~| = max(|g|, 2^-3 / s), |w~| = max(|w|, 2^(-3-k))."""
import math

import torch

import split_numerics as sn

BR, GROUP, MAX_CHUNKS, CHUNK_ROWS = 64, 5, 16, 8192
Z = sn.Z
SPLIT_INF = 131024.0            # |x| from here on splits to a non-finite low half
SUBNORMAL_ROUNDING = 2.0 ** -150


def cdiv(a, b):
    return -(-a // b)


# ---- the kernel's chunking (spconv_wgrad.cu: nchunks_of, rows_per_chunk_of) ---------------------------------------------------
def nchunks_of(m_out):
    return max(1, min(MAX_CHUNKS, cdiv(m_out, CHUNK_ROWS)))


def rows_per_chunk_of(m_out):
    return cdiv(cdiv(max(m_out, 1), nchunks_of(m_out)), BR) * BR


def chain(m_out):
    """(wgmma instructions in the longest chain, RN adds per element) of lb2_spconv_wgrad at m_out output rows"""
    stages = cdiv(min(rows_per_chunk_of(m_out), max(m_out, 1)), BR)
    return 12 * min(GROUP, stages), cdiv(stages, GROUP) + nchunks_of(m_out) - 1


def tau_h(m_out):
    n, a = chain(m_out)
    return 3.002 * 2.0 ** -22 + n * 2.0 ** -23 + a * 2.0 ** -24


def tau_s(m_out):
    n, a = chain(m_out)
    return Z * (5 * 2.0 ** -22 / math.sqrt(3) + n * 2.0 ** -23 + a * 2.0 ** -24)


def exponent(v: torch.Tensor) -> int:
    """k of the pre-scale: max|v| 2^k in [8192, 16384) over the finite elements, capped at 126; 0 when none is nonzero"""
    a = v.abs()
    m = torch.where(torch.isfinite(a), a, torch.zeros_like(a)).max().item() if v.numel() else 0.0
    if not m > 0:
        return 0
    return min(14 - math.frexp(m)[1], 126)


def split_rule(X: torch.Tensor) -> torch.Tensor:
    """X with the values the split cannot hold (|x| >= 131024) made +-inf, as the kernel's products see them"""
    return torch.where(X.abs() >= SPLIT_INF, torch.copysign(torch.full_like(X, math.inf), X), X)


# ---- weight gradient: fp64 gather-GEMM and the per-element scales ------------------------------------------------------------
def gather_gemm(X, G, nbr, kvol):
    """(kvol, X.shape[1], G.shape[1]) in X's dtype: per offset k, sum over rows o with nbr[k][o] >= 0 of X[nbr[k][o]]^T G[o]
    (nbr None: the identity, kvol 1)"""
    m = G.shape[0]
    out = torch.zeros(kvol, X.shape[1], G.shape[1], dtype=X.dtype, device=X.device)
    for k in range(kvol):
        if nbr is None:
            out[k] = X[:m].T @ G
            continue
        o = torch.nonzero(nbr[k, :m] >= 0)[:, 0]
        if o.numel():
            out[k] = X[nbr[k, o].long()].T @ G[o]
    return out


class WgradReference:
    """fp64 dW of (X, G, nbr) and the per-element scales of the model; non-finite X or G follow the split rule"""

    def __init__(self, X, G, nbr, kvol):
        self.m_out, self.kvol = G.shape[0], kvol
        self.k = exponent(G)
        X64, G64 = split_rule(X.double()), G.double()
        self.y = gather_gemm(X64, G64, nbr, kvol)
        Xa, Ga = X64.abs(), G64.abs()
        fin = lambda t: torch.where(torch.isfinite(t), t, torch.zeros_like(t))          # noqa: E731
        Xa, Ga = fin(Xa), fin(Ga)
        self.S1 = gather_gemm(Xa, Ga, nbr, kvol)
        Xf, Gf = Xa.clamp(min=2.0 ** -3), Ga.clamp(min=2.0 ** (-3 - self.k))
        self.S2f = gather_gemm(Xf ** 2, Gf ** 2, nbr, kvol)
        sg = gather_gemm(torch.ones_like(Xa[:, :1]), Ga, nbr, kvol)
        sx = gather_gemm(Xa, torch.ones_like(Ga[:, :1]), nbr, kvol)
        self.floor = 1.001 * 2.0 ** -25 * (sg + 2.0 ** -self.k * sx) + SUBNORMAL_ROUNDING
        # 65504 < |x| < 131024: hi saturates and lo = x - 65504 is no longer small, so the dropped x_lo (g s)_lo costs up to
        # |x_lo| (2^-11 |g| + 2^-25 2^-k) more (zero for every other x)
        Xe = (Xa - sn.FP16_MAX).clamp(min=0)
        self.sat = 1.001 * (2.0 ** -11 * gather_gemm(Xe, Ga, nbr, kvol) + 2.0 ** -25 * 2.0 ** -self.k
                            * gather_gemm(Xe, torch.ones_like(Ga[:, :1]), nbr, kvol)) if (Xe > 0).any() else 0.0

    def bound(self):
        return tau_h(self.m_out) * self.S1 + self.floor + self.sat

    def errors(self, dw, mask=None):
        """(max err / hard bound, max (err - saturation allowance) / sqrt(S2~)) over the elements in mask (default: all)"""
        err = (dw.double().to(self.y.device) - self.y).abs()
        h, s = err / self.bound(), (err - self.sat).clamp(min=0) / self.S2f.sqrt().clamp(min=1e-300)
        if mask is not None:
            h, s = h[mask], s[mask]
        if h.numel() == 0:
            return 0.0, 0.0
        return h.max().item(), s.max().item()


# ---- host emulation of the weight gradient's products ----------------------------------------------------------------------
SCHEMES = ("f16x3", "f16x2", "no_xlo_ghi", "unscaled")


def emulate_wgrad(X, G, nbr, kvol, scheme="f16x3"):
    """dW as the kernel forms it: the restated split of X and of G 2^k, x_hi g_hi + x_lo g_hi + x_hi g_lo per chunk of rows summed in
    fp32, the chunk partials added in chunk order in fp32, times 2^-k.  Mutants: "f16x2" holds G in one fp16 (no x_hi g_lo),
    "no_xlo_ghi" drops that cross term, "unscaled" splits G without its pre-scale."""
    if scheme not in SCHEMES:
        raise ValueError(scheme)
    m = G.shape[0]
    k = 0 if scheme == "unscaled" else exponent(G)
    xh, xl = (t.float() for t in sn.split(X))
    gh, gl = (t.float() for t in sn.split(G * 2.0 ** k))
    if scheme == "f16x2":
        gl = torch.zeros_like(gl)
    elif scheme == "no_xlo_ghi":
        xl = torch.zeros_like(xl)          # x_lo only ever multiplies g_hi
    rpc, rows = rows_per_chunk_of(m), BR * GROUP
    out = torch.zeros(kvol, X.shape[1], G.shape[1], dtype=torch.float32)
    for c in range(nchunks_of(m)):
        r0, r1 = c * rpc, min(m, (c + 1) * rpc)
        if r1 <= r0:
            continue
        part = torch.zeros_like(out)
        for kk in range(kvol):
            src = torch.arange(r0, r1) if nbr is None else nbr[kk, r0:r1].long()
            live = (src >= 0)[:, None]
            s = src.clamp(min=0)
            # one group of GROUP stages: its products summed in fp64 (the MMA chain), rounded to fp32 once, folded into the chunk's
            # fp32 total; absent rows contribute zero (the kernel zeroes both operands)
            z = lambda t: torch.where(live, t.double(), 0.0)          # noqa: E731
            a_h, a_l, b_h, b_l = z(xh[s]), z(xl[s]), z(gh[r0:r1]), z(gl[r0:r1])
            for g0 in range(0, r1 - r0, rows):
                sl = slice(g0, g0 + rows)
                acc = a_h[sl].T @ b_h[sl] + a_l[sl].T @ b_h[sl] + a_h[sl].T @ b_l[sl]
                part[kk] = part[kk] + acc.float()
        out = out + part
    return out * 2.0 ** -k


# ---- synthetic operands -------------------------------------------------------------------------------------------------------
def random_nbr(m_out, m_in, kvol, density, seed):
    """(kvol, m_out) int32 table: each entry a uniform input row with probability density, else -1"""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, max(m_in, 1), (kvol, m_out), generator=g, dtype=torch.int32)
    live = torch.rand(kvol, m_out, generator=g) < density
    return torch.where(live, idx, torch.full_like(idx, -1))


def operands(m_in, m_out, cin, cout, p, gmax, seed, col_scale=False):
    """X ~ 2^p randn (|randn| <= 1.99), G ~ randn with max|G| = gmax (and output column n times 2^e_n, e_n in -10 .. 10, the
    largest column's maximum gmax)"""
    g = torch.Generator().manual_seed(seed)
    X = (torch.randn(m_in, cin, generator=g).clamp(-1.99, 1.99) * 2.0 ** p).float()
    G = torch.randn(m_out, cout, generator=g, dtype=torch.float64)
    if col_scale:
        G = G * 2.0 ** torch.linspace(-10, 10, cout, dtype=torch.float64).round()
    if G.numel():
        G = G / G.abs().max() * gmax
    return X, G.float()


# ---- input gradient: fp64 adjoint and the forward model's scales -------------------------------------------------------------
def adjoint(G, W, nbr, m_in):
    """dX (m_in, cin) = per offset k and row o with nbr[k][o] >= 0: dX[nbr[k][o]] += G[o] W[k]^T  (nbr None: G W[0]^T); W (kvol,
    cin, cout) in G's dtype"""
    if nbr is None:
        return G @ W[0].T
    out = torch.zeros(m_in, W.shape[1], dtype=G.dtype, device=G.device)
    for k in range(W.shape[0]):
        o = torch.nonzero(nbr[k] >= 0)[:, 0]
        if o.numel():
            out.index_add_(0, nbr[k, o].long(), G[o] @ W[k].T)
    return out


def autograd_dx(G, W, nbr, m_in):
    """dX of the forward gather-GEMM y[o] = sum_k X[nbr[k][o]] W[k] (nbr None: X W[0]), by torch autograd with output gradient G"""
    X = torch.zeros(m_in, W.shape[1], dtype=G.dtype, device=G.device, requires_grad=True)
    if nbr is None:
        y = X @ W[0]
    else:
        y = torch.zeros(G.shape, dtype=G.dtype, device=G.device)
        for k in range(W.shape[0]):
            o = torch.nonzero(nbr[k] >= 0)[:, 0]
            y = y.index_add(0, o, X[nbr[k, o].long()] @ W[k])
    (dx,) = torch.autograd.grad(y, X, G)
    return dx


def input_scale_exponent(G):
    """e of _input_grad: G 2^e has its largest finite magnitude in [8192, 16384), capped at 126; 0 when no element is nonzero"""
    return exponent(G)


class DgradReference:
    """per-element scales of dX = adjoint(G, W) under the forward model of (G s, W_adj^T), unscaled by s.  cuts: the adjoint's
    output slices (the layer's input channels), each packed with its own 2^k."""

    def __init__(self, G, W, nbr, m_in, cuts):
        W = W.double()
        self.kvol, self.ctot = W.shape[0], W.shape[2]
        e = input_scale_exponent(G)
        s = 2.0 ** e
        kcol = torch.zeros(W.shape[1], dtype=torch.float64, device=W.device)
        for c0, c1 in zip(cuts[:-1], cuts[1:]):
            kcol[c0:c1] = sn.weight_exponent(W[:, c0:c1, :])
        G64 = G.double()
        self.y = autograd_dx(G64, W, nbr, m_in)
        Ga, Wa = G64.abs(), W.abs()
        Ga = torch.where(torch.isfinite(Ga), Ga, torch.zeros_like(Ga))
        self.S1 = adjoint(Ga, Wa, nbr, m_in)
        Wf = torch.maximum(Wa, 2.0 ** (-3 - kcol)[None, :, None])
        self.S2f = adjoint(Ga.clamp(min=2.0 ** -3 / s) ** 2, Wf ** 2, nbr, m_in)
        sw = adjoint(torch.ones_like(Ga), Wa, nbr, m_in)
        sg = adjoint(Ga, torch.ones_like(Wa), nbr, m_in)
        self.floor = 1.001 * 2.0 ** -25 * (sw / s + 2.0 ** -kcol * sg) + SUBNORMAL_ROUNDING

    def bounds(self):
        return sn.tau_h(self.ctot, self.kvol), sn.tau_s(self.ctot, self.kvol)

    def errors(self, dx, mask=None):
        th, _ = self.bounds()
        err = (dx.double() - self.y).abs()
        h, s = err / (th * self.S1 + self.floor), err / self.S2f.sqrt().clamp(min=1e-300)
        if mask is not None:
            h, s = h[mask], s[mask]
        return h.max().item(), s.max().item()


# ---- row sums: the sequential restatement ------------------------------------------------------------------------------------
def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """split_numerics.same_bits for fp16 / fp32 and fp64: equal bit for bit, any NaN matching any NaN"""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype != torch.float64:
        return sn.same_bits(a, b)
    na, nb = torch.isnan(a), torch.isnan(b)
    return bool(torch.equal(na, nb) and ((a.view(torch.int64) == b.view(torch.int64)) | na).all())



def sequential_segment_sum(values, order, offsets):
    """numpy: out[s] = ((+0 + v_b) + v_b+1) + ... over i in [offsets[s], offsets[s + 1]), v_i = values[order[i]], one rounding per
    add in ascending i (np.add.accumulate is that recurrence; np.sum would add pairwise)"""
    import numpy as np
    v = values if order is None else values[order]
    out = np.zeros((len(offsets) - 1, values.shape[1]), dtype=values.dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(len(offsets) - 1):
            b, e = int(offsets[s]), int(offsets[s + 1])
            if e > b:
                seg = np.concatenate([np.zeros((1, values.shape[1]), values.dtype), v[b:e]])
                out[s] = np.add.accumulate(seg, axis=0)[-1]
    return out
