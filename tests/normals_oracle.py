"""TEST INFRASTRUCTURE: a CPU restatement of open3d 0.17's `PointCloud.estimate_normals()` [o3d-mem] — numpy, vectorised over
points, fp64 throughout.  It is the specification of lidiff_b200.normals (lb2_pc_knn / lb2_pc_normals); parity against a real
open3d install is not pinned (open3d is not a dependency of this project; see DESIGN §5).

  neighbours   KDTreeSearchParamKNN(knn=30): the k_eff = min(k, n) nearest points of the cloud, the query itself included,
               ordered by (d², index) with d² = (dx·dx + dy·dy) + dz·dz, every operation rounded on its own (as pc_d2 computes it)
  covariance   open3d's one-pass cumulants (ComputeCovariance): sums of x, y, z, xx, xy, xz, yy, yz, zz in neighbour order,
               divided by the count, C = E[ppᵀ] − E[p]E[p]ᵀ; the identity when fewer than 3 neighbours
  normal       FastEigen3x3 (Geometric Tools' robust symmetric 3×3 eigensolver) for the smallest eigenvalue's eigenvector, a zero
               result replaced by (0, 0, 1), no orientation.  A covariance with a NaN or infinite entry (the cumulants overflow once
               a neighbourhood's coordinates pass ~1e154) also gives (0, 0, 1): with NaN operands the solver's comparisons pick
               branches that depend on how each maximum treats NaN, which neither open3d nor Eigen states

Every expression is evaluated in the order the C++ writes it (left to right), one rounding per operation.  The order of the three-term
dot products inside ComputeEigenvector0 is taken as ((x0·x0 + x1·x1) + x2·x2); Eigen's own reduction order is not pinned either.

It lives with the tests, not in `oracle/`: the restatements there are the recorded spec of the denoising path, from which the
committed goldens were generated, and are kept unchanged; this one specifies a post-processing step and only tests and
scripts/bench_normals.py use it.  `refined_like` is the cloud both of them measure."""
import numpy as np

TWO_THIRDS_PI = 2.09439510239319549


def refined_like(seed=0, n_base=170_000):
    """a cloud shaped like a refined completion: n_base points of two synthetic scans with 6 offsets (sigma 3 cm) around each"""
    from lidiff_b200.synth import synthetic_scan
    g = np.random.default_rng(seed)
    scan = np.concatenate([synthetic_scan(seed), synthetic_scan(seed + 1)])
    base = scan[g.choice(scan.shape[0], n_base, replace=False)]
    return (base[:, None, :] + g.normal(0.0, 0.03, (n_base, 6, 3))).reshape(-1, 3)


def d2_of(q, p):
    """pc_d2: (dx*dx + dy*dy) + dz*dz with dx = q - p per axis, every operation rounded (numpy never contracts to FMA)"""
    d = q - p
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn(points, k, spare=8):
    """(idx int64 (n, k_eff), d2 (n, k_eff)) in (d², index) order.  scipy's cKDTree proposes k_eff + spare candidates; they are
    re-ranked by the exact d² and index.  The cut is exact only when the last candidate is strictly farther than the k-th (no point
    left out can tie with or beat it); rows where it is not are searched again with twice the candidates, up to the whole cloud."""
    from scipy.spatial import cKDTree
    p = np.ascontiguousarray(points, dtype=np.float64)
    n = p.shape[0]
    ke = min(int(k), n)
    if n == 0 or ke == 0:
        return np.zeros((n, 0), np.int64), np.zeros((n, 0))
    tree = cKDTree(p)
    idx, d2 = np.zeros((n, ke), np.int64), np.zeros((n, ke))
    rows, m = np.arange(n), min(ke + spare, n)
    while rows.shape[0]:
        _, cand = tree.query(p[rows], k=m, workers=-1)
        cand = np.asarray(cand).reshape(rows.shape[0], m)
        d = d2_of(p[rows, None, :], p[cand])
        order = np.lexsort((cand, d), axis=1)                  # primary d², then index
        cand, d = np.take_along_axis(cand, order, 1), np.take_along_axis(d, order, 1)
        ok = np.ones(rows.shape[0], bool) if m == n else d[:, m - 1] > d[:, ke - 1]
        idx[rows[ok]], d2[rows[ok]] = cand[ok, :ke], d[ok, :ke]
        rows, m = rows[~ok], min(2 * m, n)
    return idx, d2


def covariances(points, idx):
    """(n, 3, 3) open3d ComputeCovariance of each row of neighbour indices (identity when fewer than 3 neighbours)"""
    p = np.asarray(points, dtype=np.float64)
    n, k = idx.shape
    cov = np.broadcast_to(np.eye(3), (n, 3, 3)).copy()
    if k < 3:
        return cov
    c = np.zeros((n, 9))
    for j in range(k):                                         # sequential sums in neighbour order
        x, y, z = (p[idx[:, j], a] for a in range(3))
        c += np.stack([x, y, z, x * x, x * y, x * z, y * y, y * z, z * z], 1)
    c /= float(k)
    cov[:, 0, 0] = c[:, 3] - c[:, 0] * c[:, 0]
    cov[:, 1, 1] = c[:, 6] - c[:, 1] * c[:, 1]
    cov[:, 2, 2] = c[:, 8] - c[:, 2] * c[:, 2]
    cov[:, 0, 1] = cov[:, 1, 0] = c[:, 4] - c[:, 0] * c[:, 1]
    cov[:, 0, 2] = cov[:, 2, 0] = c[:, 5] - c[:, 0] * c[:, 2]
    cov[:, 1, 2] = cov[:, 2, 1] = c[:, 7] - c[:, 1] * c[:, 2]
    return cov


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def _dot3(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def _ratio(a, b):
    """larger / smaller of two non-negative margins (inf when the smaller is 0 and the larger is not, 1 when both are 0)"""
    hi, lo = np.maximum(a, b), np.minimum(a, b)
    return np.where(hi == 0, 1.0, np.where(lo == 0, np.inf, hi / np.where(lo == 0, 1.0, lo)))


def _eigenvector0(A, ev):
    """ComputeEigenvector0: the largest of the three row cross products of A - ev I, normalised; + the winner / runner-up norm ratio"""
    a00, a01, a02, a11, a12, a22 = A
    r0 = np.stack([a00 - ev, a01, a02], 1)
    r1 = np.stack([a01, a11 - ev, a12], 1)
    r2 = np.stack([a02, a12, a22 - ev], 1)
    c = [_cross(r0, r1), _cross(r0, r2), _cross(r1, r2)]
    d = np.stack([_dot3(v, v) for v in c], 1)
    imax = np.zeros(d.shape[0], np.int64)
    dmax = d[:, 0].copy()
    up = d[:, 1] > dmax
    imax[up], dmax[up] = 1, d[up, 1]
    imax[d[:, 2] > dmax] = 2
    win = np.take_along_axis(d, imax[:, None], 1)[:, 0]
    runner = np.sort(d, 1)[:, 1]
    vec = np.choose(imax[:, None], c) / np.sqrt(win)[:, None]
    return vec, _ratio(np.sqrt(win), np.sqrt(runner))


def _eigenvector1(A, e0, ev1):
    """ComputeEigenvector1: the eigenvector of ev1 inside the plane orthogonal to e0; + the ratio of its closest branch decision"""
    a00, a01, a02, a11, a12, a22 = A
    n = e0.shape[0]
    pick_x = np.abs(e0[:, 0]) > np.abs(e0[:, 1])
    inv_x = 1 / np.sqrt(e0[:, 0] * e0[:, 0] + e0[:, 2] * e0[:, 2])
    inv_y = 1 / np.sqrt(e0[:, 1] * e0[:, 1] + e0[:, 2] * e0[:, 2])
    zero = np.zeros(n)
    U = np.where(pick_x[:, None], np.stack([-e0[:, 2] * inv_x, zero, e0[:, 0] * inv_x], 1),
                 np.stack([zero, e0[:, 2] * inv_y, -e0[:, 1] * inv_y], 1))
    V = _cross(e0, U)

    def amul(X):
        return np.stack([(a00 * X[:, 0] + a01 * X[:, 1]) + a02 * X[:, 2],
                         (a01 * X[:, 0] + a11 * X[:, 1]) + a12 * X[:, 2],
                         (a02 * X[:, 0] + a12 * X[:, 1]) + a22 * X[:, 2]], 1)
    AU, AV = amul(U), amul(V)
    m00 = _dot3(U, AU) - ev1
    m01 = _dot3(U, AV)
    m11 = _dot3(V, AV) - ev1
    b00, b01, b11 = np.abs(m00), np.abs(m01), np.abs(m11)
    first = b00 >= b11
    big = np.where(first, b00, b11)                            # m00 (first) or m11
    mbig = np.where(first, m00, m11)
    mx = np.maximum(big, b01)
    sub = big >= b01
    # sub: m01 /= mbig; mbig' = 1 / sqrt(1 + m01^2); m01 *= mbig'      else: mbig /= m01; m01' = 1 / sqrt(1 + mbig^2); mbig *= m01'
    with np.errstate(all="ignore"):
        t = m01 / mbig
        s_a = 1 / np.sqrt(1 + t * t)
        m01_a, mbig_a = t * s_a, s_a
        t2 = mbig / m01
        s_b = 1 / np.sqrt(1 + t2 * t2)
        m01_b, mbig_b = s_b, t2 * s_b
    m01n, mbign = np.where(sub, m01_a, m01_b), np.where(sub, mbig_a, mbig_b)
    # first: m01 * U - m00 * V      else: m11 * U - m01 * V
    cu = np.where(first, m01n, mbign)[:, None]
    cv = np.where(first, mbign, m01n)[:, None]
    vec = np.where((mx > 0)[:, None], cu * U - cv * V, U)
    margin = np.minimum(np.minimum(_ratio(np.abs(e0[:, 0]), np.abs(e0[:, 1])), _ratio(b00, b11)), _ratio(big, b01))
    return vec, margin


def fast_eigen3x3(cov):
    """open3d FastEigen3x3 of each (3, 3) covariance -> (normals (n, 3) before the zero -> (0, 0, 1) rule, diagnostics).
    Diagnostics per point: `half_det` = |half_det| (0 where the trigonometric branch is not taken: the branch on its sign),
    `cross_ratio` = winning / runner-up row cross-product norm in ComputeEigenvector0, `evec1_ratio` = the closest of
    ComputeEigenvector1's comparisons (larger / smaller; inf where it is not called).  Values near 1 (or a half_det near 0) mark
    points whose sign another rounding of acos / cos may flip."""
    cov = np.asarray(cov, dtype=np.float64)
    n = cov.shape[0]
    out = np.zeros((n, 3))
    diag = {"half_det": np.zeros(n), "cross_ratio": np.full(n, np.inf), "evec1_ratio": np.full(n, np.inf)}
    with np.errstate(all="ignore"):
        max_coeff = cov.reshape(n, 9).max(1)
        live = (max_coeff != 0) & np.isfinite(cov).all((1, 2))           # a NaN or infinite entry gives the zero vector too
        A = cov / np.where(live, max_coeff, 1.0)[:, None, None]
        a00, a01, a02, a11, a12, a22 = A[:, 0, 0], A[:, 0, 1], A[:, 0, 2], A[:, 1, 1], A[:, 1, 2], A[:, 2, 2]
        norm = (a01 * a01 + a02 * a02) + a12 * a12
        # off-diagonal zero: the axis of the smallest diagonal entry of A * max_coeff (open3d scales A back before comparing)
        c00, c11, c22 = a00 * max_coeff, a11 * max_coeff, a22 * max_coeff
        ax = np.where((c00 < c11) & (c00 < c22), 0, np.where((c11 < c00) & (c11 < c22), 1, 2))
        axis = np.eye(3)[ax]
        q = ((a00 + a11) + a22) / 3
        b00, b11, b22 = a00 - q, a11 - q, a22 - q
        p = np.sqrt((((b00 * b00 + b11 * b11) + b22 * b22) + norm * 2) / 6)
        k00 = b11 * b22 - a12 * a12
        k01 = a01 * b22 - a12 * a02
        k02 = a01 * a12 - b11 * a02
        det = ((b00 * k00 - a01 * k01) + a02 * k02) / ((p * p) * p)
        half_det = np.minimum(np.maximum(det * 0.5, -1.0), 1.0)
        angle = np.arccos(half_det) / 3.0
        beta2 = np.cos(angle) * 2
        beta0 = np.cos(angle + TWO_THIRDS_PI) * 2
        beta1 = -(beta0 + beta2)
        ev0, ev1, ev2 = q + p * beta0, q + p * beta1, q + p * beta2
        pos = half_det >= 0
        Av = (a00, a01, a02, a11, a12, a22)
        ea, cross_ratio = _eigenvector0(Av, np.where(pos, ev2, ev0))         # evec2 (pos) or evec0
        ea_min = np.where(pos, (ev2 < ev0) & (ev2 < ev1), (ev0 < ev1) & (ev0 < ev2))
        e1, evec1_ratio = _eigenvector1(Av, ea, ev1)
        e1_min = (ev1 < ev0) & (ev1 < ev2)
        last = np.where(pos[:, None], _cross(e1, ea), _cross(ea, e1))      # evec1 x evec2 (pos) or evec0 x evec1
        trig = np.where(ea_min[:, None], ea, np.where(e1_min[:, None], e1, last))
        off = norm > 0
        res = np.where(off[:, None], trig, axis)
        out = np.where(live[:, None], res, 0.0)
    t = live & off
    diag["half_det"] = np.where(t, np.abs(half_det), 0.0)
    diag["cross_ratio"] = np.where(t, cross_ratio, np.inf)
    diag["evec1_ratio"] = np.where(t & ~ea_min, evec1_ratio, np.inf)
    return out, diag


def normals_from_idx(points, idx):
    """open3d EstimateNormals given the neighbour rows: (normals (n, 3), diagnostics, covariances)"""
    cov = covariances(points, idx)
    nrm, diag = fast_eigen3x3(cov)
    zero = (nrm == 0).all(1)
    nrm[zero] = (0.0, 0.0, 1.0)
    return nrm, diag, cov


def estimate_normals(points, k=30):
    """the whole restatement: (normals (n, 3), diagnostics, covariances, idx, d2)"""
    idx, d2 = knn(points, k)
    nrm, diag, cov = normals_from_idx(points, idx)
    return nrm, diag, cov, idx, d2


def eigen_gap(cov):
    """(λ1 − λ0) / λ2 of each covariance (numpy eigvalsh, ascending); 0 where λ2 is 0"""
    w = np.linalg.eigvalsh(cov)
    with np.errstate(all="ignore"):
        return np.where(w[:, 2] > 0, (w[:, 1] - w[:, 0]) / w[:, 2], 0.0)


def clear_sign(diag, tol=1e-9):
    """points whose sign decisions all have a margin: |half_det| > tol and every compared pair apart by a factor >= 1 + tol"""
    return (diag["half_det"] > tol) & (diag["cross_ratio"] >= 1 + tol) & (diag["evec1_ratio"] >= 1 + tol)
