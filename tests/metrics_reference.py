"""TEST INFRASTRUCTURE: plain numpy restatements of what include/lidiff_b200.h promises for the evaluation-metric kernels
(csrc/metrics.cu), the yardsticks of tests/test_gpu_metrics_edges.py:

  * nearest neighbour (lb2_pc_nn): an fp64 brute force in the kernel's operation order, (dx*dx + dy*dy) + dz*dz with one rounding
    per operation and no FMA, then sqrt; lowest index on ties; only a finite d² counts, and a query without one gets (-1, +inf).
    numpy's fp64 element-wise operations are correctly rounded, as the kernel's _rn intrinsics are, so the distances are compared
    bit for bit;
  * lb2_dist_stats: the sum in the kernel's exact order (grid, per-thread strides, shared-memory tree, block partials in block
    order), numpy's (d < t).sum() counts, and the kernel's binary search (which assumes ascending thresholds) for what a raw call
    gives on other orders;
  * lb2_jsd: the same grid and order with the kernel's per-element terms, and an element-wise error bound (derived below) in place
    of bit equality, because CUDA's fp64 `log` is within 1 ulp, not correctly rounded;
  * occupancy, IoU confusion and BEV: np.histogramdd's binning as sparse int64 cell sets, never a dense grid (2048³ cells = 2^33)."""
import numpy as np

RD_THREADS = 256
RD_BLOCKS = 1024
U = 2.0 ** -53                  # unit roundoff of fp64


# ---- nearest neighbour -------------------------------------------------------------------------------------------------------
def pc_d2(q, r):
    """(len(q), len(r)) squared distances as k_pc_query forms them: (dx*dx + dy*dy) + dz*dz, every operation rounded on its own"""
    with np.errstate(invalid="ignore", over="ignore"):
        dx = q[:, None, 0] - r[None, :, 0]
        dy = q[:, None, 1] - r[None, :, 1]
        dz = q[:, None, 2] - r[None, :, 2]
        return (dx * dx + dy * dy) + dz * dz


def nn(q, r, chunk_elems=1 << 23):
    """(dist fp64, idx int64) of every query: the nearest reference point by a finite d² (lowest index on equal d²),
    dist = sqrt(d²); (+inf, -1) for a query with a non-finite coordinate or without any finite d²"""
    q, r = np.asarray(q, np.float64).reshape(-1, 3), np.asarray(r, np.float64).reshape(-1, 3)
    nq, nr = q.shape[0], r.shape[0]
    idx = np.full(nq, -1, np.int64)
    d2 = np.full(nq, np.inf)
    live = np.nonzero(np.isfinite(q).all(1))[0]
    step = max(1, chunk_elems // max(nr, 1))
    for a in range(0, live.shape[0], step):
        rows = live[a:a + step]
        d = pc_d2(q[rows], r)
        d[~(d < np.inf)] = np.inf                                   # NaN and +inf never win
        j = d.argmin(1)                                             # first minimum: the lowest index
        best = d[np.arange(rows.shape[0]), j]
        ok = best < np.inf
        idx[rows[ok]] = j[ok]
        d2[rows[ok]] = best[ok]
    return np.sqrt(d2), idx


# ---- fixed-order reductions --------------------------------------------------------------------------------------------------
def rd_blocks(n):
    """the reductions' grid: max(1, min(ceil(n / 256), 1024)) blocks of 256 threads"""
    return max(1, min(-(-int(n) // RD_THREADS), RD_BLOCKS))


def ordered_sum(v, reverse_blocks=False, drop_block=None):
    """the fp64 sum in the kernels' order: thread (b, t) adds elements b*256 + t + k*nblk*256 in increasing k from +0, each block
    reduces by the tree s[t] += s[t + o], o = 128 ... 1, and the block partials are added from +0 in block order.
    `reverse_blocks` / `drop_block` are wrong variants for the host tests.  Padding with +0 changes nothing: an accumulator that
    starts at +0 is never -0, and x + (+0) = x for every other x, NaN and inf included."""
    v = np.asarray(v, np.float64).reshape(-1)
    nblk = rd_blocks(v.shape[0])
    stride = nblk * RD_THREADS
    k = max(1, -(-v.shape[0] // stride))
    m = np.zeros(k * stride)
    m[: v.shape[0]] = v
    m = m.reshape(k, stride)
    acc = np.zeros(stride)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(k):
            acc = acc + m[i]
        s = acc.reshape(nblk, RD_THREADS).copy()
        o = RD_THREADS // 2
        while o > 0:
            s[:, :o] = s[:, :o] + s[:, o:2 * o]
            o >>= 1
    parts = [float(x) for x in s[:, 0]]
    if drop_block is not None:
        parts.pop(drop_block)
    if reverse_blocks:
        parts = parts[::-1]
    total = 0.0
    for x in parts:
        total = total + x
    return total


def path_adds(n):
    """additions an element's value passes through on its way to the result: its thread's loop, the 8 tree levels and the
    block partials (the depth used by the error bound of jsd_bound)"""
    nblk = rd_blocks(n)
    return -(-int(n) // (nblk * RD_THREADS)) + 8 + nblk


def counts_below(d, t):
    """numpy's (d < t).sum() for every threshold, in the thresholds' order (0 for a NaN threshold, as `d < nan` is all False)"""
    d, t = np.asarray(d, np.float64).reshape(-1), np.asarray(t, np.float64).reshape(-1)
    ds = np.sort(d)                                                 # NaN sorts last and is never below a threshold
    c = np.searchsorted(ds, t, side="left").astype(np.int64)
    c[np.isnan(t)] = 0
    return c


def ds_kernel_counts(d, t):
    """what k_ds_partial + k_ds_final count for thresholds in any order: each distance lands in the first k whose binary search
    (lo = 0, hi = nt; thr[mid] > v ? hi = mid : lo = mid + 1) ends at k, and counts[k] = the number landing in 0..k.  Equals
    counts_below only for ascending, NaN-free thresholds."""
    d, t = np.asarray(d, np.float64).reshape(-1), np.asarray(t, np.float64).reshape(-1)
    nt = t.shape[0]
    lo = np.zeros(d.shape[0], np.int64)
    hi = np.full(d.shape[0], nt, np.int64)
    with np.errstate(invalid="ignore"):
        while (lo < hi).any():
            act = lo < hi
            mid = (lo + hi) >> 1
            above = np.zeros(d.shape[0], bool)
            above[act] = t[mid[act]] > d[act]
            hi = np.where(act & above, mid, hi)
            lo = np.where(act & ~above, mid + 1, lo)
    return np.cumsum(np.bincount(lo, minlength=nt + 1)[:nt]).astype(np.int64)


def dist_stats(d, t):
    """(sum, counts) that lb2_dist_stats returns for ascending, NaN-free thresholds"""
    return ordered_sum(d), counts_below(d, t)


# ---- Jensen-Shannon distance -------------------------------------------------------------------------------------------------
def jsd_terms(a, b, log=np.log, drop_shared_q=False):
    """k_jsd_partial's per-element terms: t = p log(p / m), then t + q log(q / m), with p = ca / sa, q = cb / sb,
    m = (p + q) 0.5; 0 where both counts are 0 (the kernel skips those elements, and adding +0 changes no sum).
    Returns (t, |p log(p / m)| + |q log(q / m)|), the second for the error bound.  `log` and `drop_shared_q` make wrong variants."""
    a, b = np.asarray(a, np.uint32).reshape(-1), np.asarray(b, np.uint32).reshape(-1)
    sa, sb = float(int(a.sum(dtype=np.uint64))), float(int(b.sum(dtype=np.uint64)))
    with np.errstate(invalid="ignore", divide="ignore"):
        p, q = a.astype(np.float64) / sa, b.astype(np.float64) / sb
        m = (p + q) * 0.5
        tp = np.where(a > 0, p * log(p / m), 0.0)
        tq = np.where(b > 0, q * log(q / m), 0.0)
    if drop_shared_q:
        tq = np.where(a > 0, 0.0, tq)
    return np.where(a > 0, tp, 0.0) + tq, np.abs(tp) + np.abs(tq)


def jsd(a, b, **variant):
    """lb2_jsd's value from the host evaluation of its order: NaN if a histogram is empty, else sqrt(fmax(S 0.5, 0)) of the
    ordered sum S of the terms"""
    a, b = np.asarray(a, np.uint32).reshape(-1), np.asarray(b, np.uint32).reshape(-1)
    if int(a.sum(dtype=np.uint64)) == 0 or int(b.sum(dtype=np.uint64)) == 0:
        return float("nan")
    t, _ = jsd_terms(a, b, **{k: v for k, v in variant.items() if k in ("log", "drop_shared_q")})
    s = ordered_sum(t, **{k: v for k, v in variant.items() if k in ("reverse_blocks", "drop_block")})
    return float(np.sqrt(np.fmax(s * 0.5, 0.0)))


def jsd_bound(a, b):
    """(lo, hi): every value lb2_jsd may return for these histograms, from the host evaluation of its order.

    Derivation.  The kernel and jsd() perform the same operations in the same order; all but `log` are correctly rounded on both
    sides and so agree bit for bit as long as their inputs do.  CUDA's fp64 log is within 1 ulp (CUDA Programming Guide,
    double-precision functions table); take numpy's as within 1 ulp too, so the two logs L, L' of one argument differ by at most
    2 ulp(L) <= 2^-51 |L|.  With u = 2^-53 and |fl(x) - fl(y)| <= |x - y| + u |x| + u |y|:
      * a product p L: |fl(p L') - fl(p L)| <= 2^-51 |p L| + 2u |p L| (1 + 2^-51) <= 2^-50 |p L| (the same for q);
      * an element t = fl(tp + tq): |t' - t| <= e_i := 2^-50 (|tp| + |tq|) + 2u (|tp| + |tq|) (1 + 2^-50) <= 2^-49 (|tp| + |tq|);
      * every addition on an element's path (its thread's loop, the 8 tree levels, the nblk block partials: D = path_adds(n))
        adds at most u (|x| + |x'|) for its operands' sums; bounding each partial sum by the sum of the |t_i| + e_i below it,
        |S' - S| <= B := sum e_i + 2u D sum (|t_i| + e_i) (1 + 2u)^D, and (1 + 2u)^D < 1.001 for D <= 2^40.
    S 0.5 is exact, fmax(., 0) and sqrt are monotone, and the two sqrt roundings are within u each, so the kernel's value lies in
    [sqrt(fmax((S - B) 0.5, 0)) (1 - 2u), sqrt((S + B) 0.5) (1 + 2u)].  NaN (an empty histogram) is (nan, nan)."""
    a, b = np.asarray(a, np.uint32).reshape(-1), np.asarray(b, np.uint32).reshape(-1)
    if int(a.sum(dtype=np.uint64)) == 0 or int(b.sum(dtype=np.uint64)) == 0:
        return float("nan"), float("nan")
    t, mag = jsd_terms(a, b)
    s = ordered_sum(t)
    e = 2.0 ** -49 * mag
    big = float(np.sum(e)) * (1 + 1e-6) + 2 * U * path_adds(a.shape[0]) * float(np.sum(np.abs(t) + e)) * 1.001
    lo = float(np.sqrt(max((s - big) * 0.5, 0.0))) * (1 - 2 * U)
    hi = float(np.sqrt((s + big) * 0.5)) * (1 + 2 * U)
    return lo, hi


def within_jsd_bound(value, a, b):
    lo, hi = jsd_bound(a, b)
    if np.isnan(lo):
        return bool(np.isnan(value))
    return bool(lo <= value <= hi)


# ---- occupancy, confusion, BEV -------------------------------------------------------------------------------------------------
def cells(pts, edges):
    """(cell int64 per point, -1 outside the range or non-finite): np.histogramdd's bin per axis, searchsorted(edges, x, 'right')
    - 1 with the last edge in the last bin, C order (x slowest) in int64"""
    p, e = np.asarray(pts, np.float64).reshape(-1, 3), np.asarray(edges, np.float64)
    nb = e.shape[0] - 1
    b = np.searchsorted(e, p, side="right") - 1                     # NaN sorts past the last edge
    b[p == e[-1]] = nb - 1
    ok = ((b >= 0) & (b < nb)).all(1)
    b = b.astype(np.int64)
    return np.where(ok, (b[:, 0] * nb + b[:, 1]) * nb + b[:, 2], -1)


def occupancy(pts, edges):
    """(sorted occupied cells, the number of points in each, n_in)"""
    c = cells(pts, edges)
    c = c[c >= 0]
    u, n = np.unique(c, return_counts=True)
    return u, n.astype(np.int64), int(c.shape[0])


def confusion(cells_gt, cells_pred):
    """(tp, fn, fp) of two sorted cell sets"""
    tp = int(np.intersect1d(cells_gt, cells_pred, assume_unique=True).shape[0])
    return tp, int(cells_gt.shape[0]) - tp, int(cells_pred.shape[0]) - tp


def bev(cells_occ, bins):
    """(sorted nonzero columns x * bins + y, occupied z cells in each) of an occupied cell set"""
    col, n = np.unique(np.asarray(cells_occ, np.int64) // bins, return_counts=True)
    return col, n.astype(np.int64)
