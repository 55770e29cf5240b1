"""TEST INFRASTRUCTURE: restatements and the fp32 error model of the non-convolution kernels of a denoising step
(csrc/dense.cu), shared by tests/test_gpu_dense_edges.py (the kernels) and tests/test_dense_numerics_host.py (host emulations).
Nothing here imports the CUDA library.

Farthest point sampling (k_fps, k_fps_coop, k_fps_cluster): the selection SEQUENCE.  Start at point 0; every step takes the
first index of the largest running minimum of the squared distances, each computed as (dx*dx + dy*dy) + dz*dz in fp64, one
rounding per operation, left to right (no contraction).  Sorted, it is oracle.pipeline.farthest_point_sample.  `fps_sequence`
is the numpy form; `fps_sequence_torch` evaluates the same operations one torch op each (no fusion, so no contraction; torch's
argmax returns the first maximal index) on any device, for many scans at once.

Nearest neighbour (k_nn_match, k_nn_match_tree): per query the key of least exact int64 squared distance, plus 2^62 when the
batches differ (k_nn_match with batch_scale 0; the tree kernel's rule), lowest key index on ties.

Error model of the dense layers, u = 2^-24, gamma_n = n u / (1 - n u), slope = float32(0.1):
  * k_linear, per output element: one fp32 FMA chain over k = 0 .. n_in-1 from +0 (n_in roundings), then + b, then + addend
    (one rounding each), then the activation.  A recursive sum with m roundings is within gamma_m of the sum of the absolute
    values of its terms, so with S = sum_k |x'_k w_k| + |b| + |addend|
        |v - v64| <= gamma_(n_in + 2) S.
    With prebias, x'_k = pre_act(x_k + p_k) costs one rounding for the add and one for the slope multiply:
        |v - v64| <= gamma_(n_in + 4) S.
  * k_head_mlp, per row: hidden unit j is four lanes' FMA chains of n_in / 4 terms each, two butterfly adds and + b0, so every
    term passes through n_in / 4 + 3 roundings:  E_h <= gamma_(n_in/4 + 3) (sum_k |x_k w0_jk| + |b0_j|).  The leaky ReLU is
    1-Lipschitz and rounds once when its input is negative:  E_a <= E_h + u slope (|h| + E_h).  Output c is an FMA chain over
    n_hid and + b1:
        E_o <= sum_j |w1_cj| E_a_j + gamma_(n_hid + 1) (sum_j |w1_cj| (|a_j| + E_a_j) + |b1_c|).
  * Activations of the output: none adds nothing; the leaky ReLU adds u slope (|v| + E); tanhf is 1-Lipschitz and within
    2 ulp of tanh (CUDA C++ Programming Guide, "Mathematical Functions", single-precision table: tanhf(x), 2 ulp), so it adds
    2^-22 (|tanh v| + E) + 2^-148.
  * The fp64 reference itself is within gamma64_m of the same S (2^-53 per operation); it is added to each bound.
Every term is a bound on a rounding the kernel performs; nothing is fitted to measured errors."""
import math

import numpy as np

U = 2.0 ** -24
U64 = 2.0 ** -53
SLOPE = float(np.float32(0.1))           # the kernels' 0.1f
TANH_ULP = 2                            # tanhf, CUDA C++ Programming Guide single-precision table


def gamma(n, u=U):
    return n * u / (1.0 - n * u)


# ---- farthest point sampling ------------------------------------------------------------------------------------------------
def fps_sequence(points, n_samples):
    """numpy: the indices in the order they are selected"""
    p = np.asarray(points, dtype=np.float64)
    dist = np.full(p.shape[0], np.inf)
    seq = np.empty(n_samples, dtype=np.int64)
    cur = 0
    for i in range(n_samples):
        seq[i] = cur
        dx, dy, dz = p[:, 0] - p[cur, 0], p[:, 1] - p[cur, 1], p[:, 2] - p[cur, 2]
        d = (dx * dx + dy * dy) + dz * dz
        np.minimum(dist, d, out=dist)
        cur = int(np.argmax(dist))
    return seq


def fps_sequence_torch(scans, n_samples):
    """torch fp64, one op per kernel: (len(scans), n_samples) int64 selection sequences of the (n_b, 3) tensors `scans`, all on
    one device; padding rows carry -inf and can never win"""
    import torch
    dev = scans[0].device
    B, N = len(scans), max(int(s.shape[0]) for s in scans)
    P = torch.zeros(B, N, 3, dtype=torch.float64, device=dev)
    dist = torch.full((B, N), -math.inf, dtype=torch.float64, device=dev)
    for b, s in enumerate(scans):
        P[b, : s.shape[0]] = s.to(torch.float64)
        dist[b, : s.shape[0]] = math.inf
    px, py, pz = P[..., 0].contiguous(), P[..., 1].contiguous(), P[..., 2].contiguous()
    rows = torch.arange(B, device=dev)
    cur = torch.zeros(B, dtype=torch.int64, device=dev)
    seq = torch.empty(B, n_samples, dtype=torch.int64, device=dev)
    for i in range(n_samples):
        seq[:, i] = cur
        dx = px - px[rows, cur][:, None]
        dy = py - py[rows, cur][:, None]
        dz = pz - pz[rows, cur][:, None]
        d = torch.add(torch.add(torch.mul(dx, dx), torch.mul(dy, dy)), torch.mul(dz, dz))
        dist = torch.minimum(dist, d)
        cur = torch.argmax(dist, dim=1)
    return seq


# ---- nearest neighbour ------------------------------------------------------------------------------------------------------
BATCH_PENALTY = 1 << 62


def nn_brute(q, k, chunk=2048):
    """q (nq, 4), k (nk, 4) integer [b, x, y, z]: index of the nearest key, exact int64, +2^62 across batches, lowest index on ties"""
    q, k = np.asarray(q, dtype=np.int64), np.asarray(k, dtype=np.int64)
    out = np.empty(q.shape[0], dtype=np.int64)
    for s in range(0, q.shape[0], chunk):
        qq = q[s:s + chunk, None, :]
        d = ((qq[..., 1] - k[None, :, 1]) ** 2 + (qq[..., 2] - k[None, :, 2]) ** 2 + (qq[..., 3] - k[None, :, 3]) ** 2)
        d = d + np.where(qq[..., 0] != k[None, :, 0], BATCH_PENALTY, 0)
        out[s:s + chunk] = np.argmin(d, axis=1)
    return out


# ---- dense layers: fp64 references and bounds ---------------------------------------------------------------------------------
def _act64(v, act):
    if act == 1:
        return np.where(v > 0, v, SLOPE * v)
    if act == 2:
        return np.tanh(v)
    return v


def _act_bound(v, e, act):
    """bound after the output activation, from the fp64 pre-activation v and its bound e"""
    if act == 1:
        return e + U * SLOPE * (np.abs(v) + e)
    if act == 2:
        return e + TANH_ULP * 2.0 ** -23 * (np.abs(np.tanh(v)) + e) + 2.0 ** -148
    return e


def linear_reference(x, w, b=None, addend=None, act=0, prebias=None, pre_act=0):
    """(y64, bound) of lb2_linear: x (m, n_in), w (n_out, n_in), b (n_out), addend (m, n_out), all fp32 arrays"""
    x, w = x.astype(np.float64), w.astype(np.float64)
    n_in = x.shape[1]
    xp = _act64(x + prebias.astype(np.float64), pre_act) if prebias is not None else x
    v = xp @ w.T
    S = np.abs(xp) @ np.abs(w).T
    if b is not None:
        v, S = v + b.astype(np.float64), S + np.abs(b.astype(np.float64))
    if addend is not None:
        v, S = v + addend.astype(np.float64), S + np.abs(addend.astype(np.float64))
    m = n_in + (4 if prebias is not None else 2)
    e = (gamma(m) + gamma(m, U64)) * S
    return _act64(v, act), _act_bound(v, e, act)


def head_mlp_reference(x, w0, b0, w1, b1, out_act=0):
    """(y64, bound) of lb2_head_mlp: x (m, n_in), w0 (n_hid, n_in), b0 (n_hid), w1 (n_out, n_hid), b1 (n_out)"""
    x, w0, b0, w1, b1 = (a.astype(np.float64) for a in (x, w0, b0, w1, b1))
    n_in, n_hid = w0.shape[1], w0.shape[0]
    h = x @ w0.T + b0
    Sh = np.abs(x) @ np.abs(w0).T + np.abs(b0)
    eh = (gamma(n_in // 4 + 3) + gamma(n_in + 1, U64)) * Sh
    a = np.where(h > 0, h, SLOPE * h)
    ea = eh + U * SLOPE * (np.abs(h) + eh)
    v = a @ w1.T + b1
    eo = ea @ np.abs(w1).T + (gamma(n_hid + 1) + gamma(n_hid + 1, U64)) * ((np.abs(a) + ea) @ np.abs(w1).T + np.abs(b1))
    return _act64(v, out_act), _act_bound(v, eo, out_act)


def within(y, ref, bound):
    """max over elements of |y - ref| / bound (0 where both are 0); NaN anywhere in y counts as infinitely far"""
    y = np.asarray(y, dtype=np.float64)
    err = np.abs(y - ref)
    err = np.where(np.isnan(err), np.inf, err)
    r = np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 1e-300))
    return float(r.max()) if r.size else 0.0


# ---- host emulations of the kernels' fp32 order (and mutants of it) ------------------------------------------------------------
def _fma32(a, b, c):
    """fp32 FMA through fp64: a*b is exact in fp64, the add rounds at 2^-53 before the fp32 rounding (within the model's slack)"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def tf32(a):
    """round fp32 to the 10-bit mantissa of TF32 (nearest, ties away), as a tensor core would read it"""
    i = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    i = ((i + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return i.view(np.float32)


def emulate_linear(x, w, b=None, addend=None, act=0, prebias=None, pre_act=0, mutant=None):
    """k_linear in numpy fp32: the FMA chain over k in ascending order, + b, + addend, the activation.  mutant "tf32" rounds both
    operands to TF32; "drop_tile" leaves out the last k-tile of 16 (the partial one when n_in % 16 != 0)"""
    x, w = x.astype(np.float32), w.astype(np.float32)
    n_in = x.shape[1]
    if prebias is not None:
        s = (x + prebias.astype(np.float32)).astype(np.float32)
        x = np.where(s > 0, s, np.float32(0.1) * s).astype(np.float32) if pre_act == 1 else s
    if mutant == "tf32":
        x, w = tf32(x), tf32(w)
    k_end = 16 * ((n_in - 1) // 16) if mutant == "drop_tile" else n_in
    acc = np.zeros((x.shape[0], w.shape[0]), dtype=np.float32)
    for k in range(k_end):
        acc = _fma32(x[:, k:k + 1], w[None, :, k], acc)
    if b is not None:
        acc = (acc + b.astype(np.float32)).astype(np.float32)
    if addend is not None:
        acc = (acc + addend.astype(np.float32)).astype(np.float32)
    return _act32(acc, act)


def _act32(v, act):
    if act == 1:
        return np.where(v > 0, v, np.float32(0.1) * v).astype(np.float32)
    if act == 2:
        return np.tanh(v.astype(np.float64)).astype(np.float32)       # correctly rounded: inside tanhf's 2 ulp
    return v


def emulate_head_mlp(x, w0, b0, w1, b1, out_act=0, mutant=None):
    """k_head_mlp in numpy fp32: lane q sums the input channels k*16 + q*4 .. +3 (k ascending) by FMA, the butterfly
    (s0 + s1) + (s2 + s3), + b0, the leaky ReLU, the FMA chain over the hidden units, + b1, the activation.  mutant "tf32" rounds
    x, w0 and w1 to TF32; "drop_hidden" leaves out the last hidden unit"""
    x, w0, b0, w1, b1 = (a.astype(np.float32) for a in (x, w0, b0, w1, b1))
    if mutant == "tf32":
        x, w0, w1 = tf32(x), tf32(w0), tf32(w1)
    m, n_in = x.shape
    n_hid, n_out = w0.shape[0], w1.shape[0]
    nk = n_in // 16
    xs, ws = x.reshape(m, nk, 4, 4), w0.reshape(n_hid, nk, 4, 4)          # [row, 64-byte piece k, lane q, element e]
    lanes = np.zeros((m, n_hid, 4), dtype=np.float32)                     # lane q's chain, every hidden unit at once
    for k in range(nk):
        for e in range(4):
            lanes = _fma32(xs[:, None, k, :, e], ws[None, :, k, :, e], lanes)
    h = ((lanes[..., 0] + lanes[..., 1]).astype(np.float32) + (lanes[..., 2] + lanes[..., 3]).astype(np.float32)).astype(np.float32)
    h = (h + b0).astype(np.float32)
    h = np.where(h > 0, h, np.float32(0.1) * h).astype(np.float32)
    o = np.zeros((m, n_out), dtype=np.float32)
    for j in range(n_hid - (1 if mutant == "drop_hidden" else 0)):
        o = _fma32(w1[None, :, j], h[:, j:j + 1], o)
    return _act32((o + b1).astype(np.float32), out_act)
