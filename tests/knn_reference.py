"""TEST INFRASTRUCTURE: a plain fp64 brute force of the exact self-k-nearest-neighbour contract (lb2_pc_knn), and a numpy emulation
of the order in which lb2_pc_tree_build lays the cloud out (csrc/metrics.cu), the yardsticks of tests/test_gpu_knn_normals_edges.py.

  * `knn(points, k, rows=None)`: for every row, the k_eff = min(k, n) points of the cloud with the smallest finite
    d² = (dx·dx + dy·dy) + dz·dz (normals_oracle.d2_of: one rounding per operation, no FMA), ordered by (d², index); the slots
    nothing fills hold (-1, +inf), and a row with a NaN or infinite coordinate has only such slots.  No k-d tree is involved:
    scipy's cKDTree has its own overflow, underflow and NaN behaviour, so it cannot be the reference at those edges.
  * `tree_layout(points)`: the tree's bounding box, 10-bit Morton codes and stable sort, as k_pc_bbox / k_pc_morton / rs_sort_keys
    compute them (`fixed=False` restates the build before rows with a non-finite coordinate were kept out of it).  The host tests
    use it to show that a cloud really puts the points tying with the k-th neighbour in other leaves than the query's and outside
    the 32 sorted neighbours that seed k_pc_knn's list; the GPU tests check that the tree a build leaves has this order.
  * the clouds both of them use: lattices, magnitudes where fp32 node boxes are coarse or leave the fp32 range, squared distances
    that overflow or underflow, signed zeros, duplicate groups longer than the seed window."""
import numpy as np

from normals_oracle import d2_of

PC_LEAF = 8
PC_BITS = 10
SEED = 32                       # k_pc_knn seeds its list with the 32 points around the query in the sorted order


# ---- brute force -------------------------------------------------------------------------------------------------------------
def _d2_rows(q, px, py, pz):
    """d2_of(q[:, None], p[None]) with the same operations in the same order, in place on (m, n) arrays"""
    d = np.subtract(q[:, 0, None], px)
    d *= d
    t = np.subtract(q[:, 1, None], py)
    t *= t
    d += t
    np.subtract(q[:, 2, None], pz, out=t)
    t *= t
    d += t
    return d


def knn(points, k, rows=None, chunk_elems=1 << 22):
    """(idx int64 (m, k_eff), d2 fp64 (m, k_eff)) of `rows` (default: every point), k_eff = min(k, n)"""
    p = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    n = p.shape[0]
    ke = min(int(k), n)
    rows = np.arange(n) if rows is None else np.asarray(rows, np.int64).reshape(-1)
    idx = np.full((rows.shape[0], ke), -1, np.int64)
    d2 = np.full((rows.shape[0], ke), np.inf)
    if ke == 0:
        return idx, d2
    live = np.isfinite(p).all(1)
    px, py, pz = (np.ascontiguousarray(p[:, a]) for a in range(3))
    step = max(1, chunk_elems // n)
    for a in range(0, rows.shape[0], step):
        r = rows[a:a + step]
        with np.errstate(invalid="ignore", over="ignore", under="ignore"):
            d = _d2_rows(p[r], px, py, pz)
        d[~(d < np.inf)] = np.inf                                   # NaN and +inf never enter a list
        d[~live[r]] = np.inf                                        # a non-finite point has no neighbours
        kth = np.partition(d, ke - 1, axis=1)[:, ke - 1]
        less = d < kth[:, None]
        eq = d == kth[:, None]
        need = ke - less.sum(1)
        tied = eq.sum(1) > need
        take = less | eq
        if tied.any():                                              # the lowest indices among the points at the k-th d²
            take[tied] = less[tied] | (eq[tied] & (np.cumsum(eq[tied], 1) <= need[tied, None]))
        cc = np.nonzero(take)[1].reshape(r.shape[0], ke)            # ascending index within a row
        dd = np.take_along_axis(d, cc, 1)
        o = np.argsort(dd, axis=1, kind="stable")                   # (d², index)
        cc, dd = np.take_along_axis(cc, o, 1), np.take_along_axis(dd, o, 1)
        cc[dd == np.inf] = -1
        idx[a:a + step], d2[a:a + step] = cc, dd
    return idx, d2


# ---- the tree's layout -------------------------------------------------------------------------------------------------------
def okey(v):
    """pc_okey: fp64 bits as uint64 keys with the same order (a NaN with the sign bit set below -inf, one without above +inf)"""
    u = np.ascontiguousarray(v, np.float64).view(np.uint64)
    return np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))


def unkey(k):
    k = np.asarray(k, np.uint64)
    return np.where(k >> np.uint64(63), k & np.uint64(0x7fffffffffffffff), ~k).astype(np.uint64).view(np.float64)


def _spread10(v):
    v = v.astype(np.uint32) & np.uint32(0x3ff)
    for s, m in ((16, 0x030000ff), (8, 0x0300f00f), (4, 0x030c30c3), (2, 0x09249249)):
        v = (v | (v << np.uint32(s))) & np.uint32(m)
    return v


def bbox(points, fixed=True):
    """(lo (3,), hi (3,)) of k_pc_bbox: over the rows with three finite coordinates (fixed), or every coordinate by its key"""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    if fixed:
        p = p[np.isfinite(p).all(1)]
    if p.shape[0] == 0:
        return unkey(np.full(3, ~np.uint64(0))), unkey(np.zeros(3, np.uint64))
    k = okey(p)
    return unkey(k.min(0)), unkey(k.max(0))


def morton(points, lo, hi, fixed=True):
    """k_pc_morton's codes (uint32) in the grid over [lo, hi]; a row with a non-finite coordinate gets 1 << 30 (fixed)"""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        ext = 0.0
        for a in range(3):
            ext = np.fmax(ext, hi[a] - lo[a])
        scale = (2 ** PC_BITS - 1) / ext if ext > 0 else 0.0
        c = np.fmin(np.fmax((p - lo) * scale, 0.0), float(2 ** PC_BITS - 1)).astype(np.uint32)
    code = _spread10(c[:, 0]) | (_spread10(c[:, 1]) << np.uint32(1)) | (_spread10(c[:, 2]) << np.uint32(2))
    if fixed:
        code[~np.isfinite(p).all(1)] = np.uint32(1 << (3 * PC_BITS))
    return code


def tree_layout(points, fixed=True):
    """dict(lo, hi, codes, order): order[s] = the point in sorted slot s (a stable sort of the codes)"""
    lo, hi = bbox(points, fixed)
    codes = morton(points, lo, hi, fixed)
    return {"lo": lo, "hi": hi, "codes": codes, "order": np.argsort(codes, kind="stable")}


def seed_window(slot, n):
    """[a0, a0 + 32) sorted slots k_pc_knn measures first for the point in `slot`"""
    a0 = np.clip(np.asarray(slot) - SEED // 2, 0, n - SEED) if n >= SEED else np.zeros_like(slot)
    return a0, a0 + min(SEED, n)


def ties_outside(points, k, rows, layout=None):
    """(n_tied (m,), n_outside (m,)) for each of `rows`: n_tied = the number of points at exactly the row's k-th d² (0 where that
    slot is empty), n_outside = those of them in another leaf than the query's and outside its seed window"""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    n = p.shape[0]
    lay = tree_layout(p) if layout is None else layout
    slot = np.empty(n, np.int64)
    slot[lay["order"]] = np.arange(n)
    _, d2 = knn(p, k, rows)
    kth = d2[:, -1]
    n_tied, n_out = np.zeros(len(rows), np.int64), np.zeros(len(rows), np.int64)
    for m, r in enumerate(rows):
        if not np.isfinite(kth[m]):
            continue
        with np.errstate(all="ignore"):
            at = np.nonzero(d2_of(p[r], p) == kth[m])[0]
        s = slot[at]
        a0, a1 = seed_window(slot[r], n)
        out = (s // PC_LEAF != slot[r] // PC_LEAF) & ((s < a0) | (s >= a1))
        n_tied[m], n_out[m] = at.shape[0], int(out.sum())
    return n_tied, n_out


# ---- clouds ------------------------------------------------------------------------------------------------------------------
def lattice(m, spacing, g, origin=(0.0, 0.0, 0.0)):
    """an m³ lattice, permuted so that index order is not spatial order"""
    ax = np.arange(m) * spacing
    lat = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3) + np.asarray(origin)
    return lat[g.permutation(lat.shape[0])]


def lattice_offset(g):
    ax = np.arange(24) * 2.0 ** -10
    lat = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    lat = lat + g.uniform(-2.0 ** -13, 2.0 ** -13, lat.shape) + np.array([1e6, -1e6, 1e7])
    return lat[g.permutation(lat.shape[0])]


def huge(g, scale, n=3000):
    s = g.choice([-1.0, 1.0], (n, 3))
    return s * scale * g.uniform(1, 2, (n, 3))


def duplicate_groups(g, size, groups):
    """`groups` distinct points, each repeated `size` times, shuffled"""
    p = np.repeat(g.uniform(-5, 5, (groups, 3)), size, 0)
    return p[g.permutation(p.shape[0])]


def overflow(g, scale, n=1500):
    """points of norm ~scale in random directions, with 40 near-duplicates (relative offsets ~1e-12) of the first 40 and 20 exact
    copies of the next 20"""
    u = g.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = u * scale
    near = p[:40] * (1 + g.uniform(-1e-12, 1e-12, (40, 3)))
    q = np.concatenate([p, near, p[40:60]])
    return q[g.permutation(q.shape[0])]


def _signed_zero(g):
    z = np.array([[0.0, 0.0, 0.0], [-0.0, 0.0, -0.0], [-0.0, -0.0, -0.0], [0.0, -0.0, 0.0]] * 5)
    return np.concatenate([g.normal(0, 1.0, (500, 3)), z])[::-1].copy()


KNN_CLOUDS = {
    # integer and dyadic lattices: at k = 8 the k-th slot falls in the 12-point d² = 2 shell, so the index decides across boxes
    "z3": lambda g: lattice(14, 1.0, g, (3.0, -7.0, 11.0)),
    "dyadic": lambda g: lattice(14, 2.0 ** -10, g, (0.5, -0.25, 2.0)),
    "lattice_offset": lattice_offset,                                 # a 2⁻¹⁰ lattice at 1e6 / 1e7: coarse fp32 node boxes
    "pm_1e39": lambda g: huge(g, 1e39),                               # node boxes outside the fp32 range
    "pm_1e300": lambda g: huge(g, 1e300),
    "mixed_magnitudes": lambda g: np.concatenate([huge(g, 1e39, 1000), g.normal(0, 10, (1000, 3)), huge(g, 1e300, 1000)]),
    "subnormal": lambda g: g.uniform(-1, 1, (4000, 3)) * 1e-310,      # every d² underflows to 0
    "subnormal_d2": lambda g: g.uniform(-1, 1, (4000, 3)) * 1e-156,
    "signed_zero": _signed_zero,
    "line_and_outlier": lambda g: np.concatenate([np.stack([g.uniform(0, 1e-12, 3000), np.zeros(3000), np.zeros(3000)], 1),
                                                  [[1e5, 1e5, 1e5]]])[g.permutation(3001)],
    "overflow_1e150": lambda g: overflow(g, 1e150),                   # d² ~1e300: exact
    "overflow_1e200": lambda g: overflow(g, 1e200),                   # every d² overflows except those to exact copies
    "dup50": lambda g: duplicate_groups(g, 50, 60),                   # groups longer than the seed window
    "dup200": lambda g: duplicate_groups(g, 200, 15),
    "identical_20000": lambda g: np.full((20_000, 3), -1.75),
}

# clouds whose k-th slot ties must reach past the query's leaf and its seed window (tests/test_knn_reference_host.py)
TIE_CLOUDS = ("z3", "dyadic", "subnormal", "dup50", "dup200", "identical_20000")


def cloud(name):
    return KNN_CLOUDS[name](np.random.default_rng(sum(map(ord, name))))
