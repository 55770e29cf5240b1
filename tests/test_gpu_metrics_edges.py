"""The evaluation-metric kernels (csrc/metrics.cu) at their edges, against the restatements of tests/metrics_reference.py:
  * lb2_pc_tree_build + lb2_pc_nn bit for bit (distance and index): non-finite queries and reference points, squared distances
    at the overflow edge, magnitudes where the fp32 node boxes are coarse or leave the fp32 range, subnormals, signed zeros,
    degenerate Morton grids and the leaf-padding edge;
  * metrics.chamfer_distance with a NaN or infinite row: a non-finite loss, a backward that completes, and the finite rows' terms
    unchanged;
  * lb2_dist_stats: the sum bit for bit where the grid changes shape, the strict `<` at and one ulp around each threshold,
    duplicate thresholds, the threshold-count limits, non-finite distances, and evaluate_scan with thresholds in any order;
  * lb2_jsd within the restatement's error bound, exact 0 for identical histograms, sqrt(ln 2) for disjoint ones, NaN for empty
    ones, and totals that need 64 bits;
  * lb2_voxel_occupancy, lb2_occupancy_confusion and lb2_occupancy_bev against sparse cell sets, up to 2048³ = 2^33 cells."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import metrics_reference as mr
from lidiff_b200 import metrics as M

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def h():
    from lidiff_b200 import _lib
    return _lib.get_handle(DEV)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


# ---- nearest neighbour -------------------------------------------------------------------------------------------------------
def gpu_nn(h, q, r):
    """lb2_pc_nn's raw (dist, idx): the index is read as the kernel wrote it, nothing is gathered with it"""
    qt = torch.as_tensor(np.ascontiguousarray(q, np.float64), device=DEV)
    rt = torch.as_tensor(np.ascontiguousarray(r, np.float64), device=DEV)
    dist = torch.full((qt.shape[0],), -7.0, dtype=torch.float64, device=DEV)
    idx = torch.full((qt.shape[0],), -7, dtype=torch.int32, device=DEV)
    h.pc_nn(qt, h.pc_tree(rt), dist, idx)
    return dist.cpu().numpy(), idx.cpu().numpy().astype(np.int64)


def check_nn(h, q, r, rows=None):
    """the GPU's distances and indices equal the restatement's bit for bit (on `rows` of q only, when given)"""
    d, j = gpu_nn(h, q, r)
    if rows is not None:
        q, d, j = q[rows], d[rows], j[rows]
    wd, wj = mr.nn(q, r)
    bad = np.nonzero((j != wj) | ~(d.view(np.int64) == wd.view(np.int64)))[0]
    assert bad.shape[0] == 0, f"{bad.shape[0]} queries differ, first {bad[:4]}: gpu {d[bad[:4]]} {j[bad[:4]]}, want {wd[bad[:4]]} {wj[bad[:4]]}"
    return d, j


def gauss(n, seed, spread=10.0):
    return np.random.default_rng(seed).normal(0, spread, (n, 3))


def _nonfinite_rows(g, n, values=(np.nan, np.inf, -np.inf)):
    """n rows, each with one non-finite coordinate or all three"""
    p = g.normal(0, 10, (n, 3))
    for i in range(n):
        v = values[i % len(values)]
        if (i // len(values)) % 4 == 3:
            p[i] = v
        else:
            p[i, (i // len(values)) % 4 % 3] = v
    return p


def test_nn_non_finite_queries_give_minus_one(h):
    g = np.random.default_rng(0)
    r = gauss(5000, 1)
    q = np.concatenate([g.normal(0, 12, (2000, 3)), _nonfinite_rows(g, 300)])
    q = q[g.permutation(q.shape[0])]
    d, j = check_nn(h, q, r)
    bad = ~np.isfinite(q).all(1)
    assert (j[bad] == -1).all() and (d[bad] == np.inf).all() and (j[~bad] >= 0).all()
    d0, j0 = gpu_nn(h, q[~bad], r)                                  # the finite queries keep their bits
    assert same_bits(d[~bad], d0) and np.array_equal(j[~bad], j0)


def test_nn_non_finite_reference_points_are_nobodys_neighbour(h):
    g = np.random.default_rng(2)
    r = np.concatenate([gauss(3000, 3), _nonfinite_rows(g, 200)])
    perm = g.permutation(r.shape[0])
    r = r[perm]
    q = g.normal(0, 12, (2500, 3))
    d, j = check_nn(h, q, r)
    live = np.nonzero(np.isfinite(r).all(1))[0]
    d0, j0 = gpu_nn(h, q, r[live])                                  # the finite sub-cloud's answer, in the original indices
    assert same_bits(d, d0) and np.array_equal(j, live[j0])


def test_nn_reference_without_a_finite_point(h):
    g = np.random.default_rng(4)
    q = np.concatenate([g.normal(0, 5, (500, 3)), _nonfinite_rows(g, 30)])
    for r in (_nonfinite_rows(g, 1), _nonfinite_rows(g, 77), np.full((9, 3), np.nan)):
        d, j = gpu_nn(h, q, r)
        assert (j == -1).all() and (d == np.inf).all()


def test_nn_squared_distances_at_the_overflow_edge(h):
    g = np.random.default_rng(5)
    r = np.concatenate([gauss(2000, 6), g.normal(0, 1, (50, 3)) * 1e150])
    unit = g.normal(size=(600, 3))
    unit /= np.linalg.norm(unit, axis=1, keepdims=True)
    q150, q200 = unit[:300] * 1e150, unit[300:] * 1e200
    d, j = check_nn(h, np.concatenate([q150, q200, g.normal(0, 10, (300, 3))]), r)
    assert (j[:300] >= 0).all() and np.isfinite(d[:300]).all()
    assert (j[300:600] == -1).all() and (d[300:600] == np.inf).all()


def _lattice_offset(g):
    ax = np.arange(24) * 2.0 ** -10
    lat = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    lat = lat + g.uniform(-2.0 ** -13, 2.0 ** -13, lat.shape) + np.array([1e6, -1e6, 1e7])
    return lat[g.permutation(lat.shape[0])]


def _huge(g, scale):
    s = g.choice([-1.0, 1.0], (3000, 3))
    return s * scale * g.uniform(1, 2, (3000, 3))


NN_CLOUDS = {
    # (reference, queries) builders
    "lattice_offset": lambda g: (_lattice_offset(g), _lattice_offset(g)[:3000] + g.normal(0, 2.0 ** -11, (3000, 3))),
    "pm_1e39": lambda g: (_huge(g, 1e39), _huge(g, 1e39) * 1.0000001),
    "pm_1e300": lambda g: (_huge(g, 1e300), np.concatenate([_huge(g, 1e300), _huge(g, 1e39)[:500], g.normal(size=(500, 3))])),
    "mixed_magnitudes": lambda g: (np.concatenate([_huge(g, 1e39)[:1000], gauss(1000, 7), _huge(g, 1e300)[:1000]]),
                                   np.concatenate([_huge(g, 1e39)[:700], gauss(700, 8), _huge(g, 1e300)[:700]])),
    # every d² underflows to 0: all points tie and the walk must reach index 0 through the whole tree
    "subnormal": lambda g: (g.uniform(-1, 1, (4000, 3)) * 1e-310, g.uniform(-1.5, 1.5, (3000, 3)) * 1e-310),
    "subnormal_d2": lambda g: (g.uniform(-1, 1, (4000, 3)) * 1e-156, g.uniform(-1.5, 1.5, (3000, 3)) * 1e-156),
    "signed_zero": lambda g: (np.concatenate([gauss(500, 9, 1.0), [[0.0, 0.0, 0.0], [-0.0, 0.0, -0.0], [-0.0, -0.0, -0.0],
                                                                    [0.0, -0.0, 0.0]] * 5])[::-1].copy(),
                              np.array([[0.0, 0.0, 0.0], [-0.0, -0.0, -0.0], [-0.0, 0.0, 0.0], [1e-320, -1e-320, 0.0]] * 3)),
    "identical_100k": lambda g: (np.full((100_000, 3), 3.25), g.normal(0, 5, (500, 3))),
    "line_and_outlier": lambda g: (np.concatenate([np.stack([g.uniform(0, 1e-12, 20_000), np.zeros(20_000), np.zeros(20_000)], 1),
                                                   [[1e5, 1e5, 1e5]]])[g.permutation(20_001)],
                                   np.concatenate([g.uniform(-1e-12, 2e-12, (1500, 3)), g.normal(1e5, 1.0, (500, 3)),
                                                   g.normal(0, 1e3, (500, 3))])),
}


@pytest.mark.parametrize("case", list(NN_CLOUDS))
def test_nn_bit_exact_at_magnitude_and_degenerate_edges(h, case):
    g = np.random.default_rng(len(case))
    r, q = NN_CLOUDS[case](g)
    d, j = check_nn(h, q, r)
    if case == "identical_100k":
        assert (j == 0).all()
    if case == "signed_zero":
        assert (j == np.nonzero((r == 0).all(1))[0][0]).all() and (d == 0).all()


@pytest.mark.parametrize("n_ref", [1_048_576, 1_048_577])
def test_nn_leaf_padding_edge(h, n_ref):
    """2^17 full leaves, and one point more: twice the leaves, most of them empty"""
    g = np.random.default_rng(n_ref)
    r = g.normal(0, 20, (n_ref, 3))
    q = np.concatenate([r[g.integers(0, n_ref, 2000)] + g.normal(0, 0.01, (2000, 3)), g.normal(0, 30, (2000, 3)), r[-5:]])
    d, j = gpu_nn(h, q, r)
    kd, _ = cKDTree(r).query(q)
    assert np.abs(d - kd).max() <= 1e-12 * max(1.0, kd.max())
    rows = np.concatenate([g.choice(q.shape[0] - 5, 250, replace=False), np.arange(q.shape[0] - 5, q.shape[0])])
    check_nn(h, q, r, rows=rows)
    assert np.array_equal(j[-5:], np.arange(n_ref - 5, n_ref))


# ---- Chamfer loss with a non-finite row --------------------------------------------------------------------------------------
@pytest.mark.parametrize("cloud", ["x", "y"])
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_chamfer_with_a_non_finite_row(cloud, value):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 3000, 3, generator=g).to(DEV)
    y = (torch.randn(1, 2500, 3, generator=g) * 1.1).to(DEV)
    bad_row = 17
    src = x if cloud == "x" else y
    src[0, bad_row, 1] = float(value)
    xx, yy = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    loss, _ = M.chamfer_distance(xx, yy)
    assert not torch.isfinite(loss)
    loss.backward()
    torch.cuda.synchronize()
    assert xx.grad is not None and yy.grad is not None
    keep = torch.ones(src.shape[1], dtype=torch.bool, device=DEV)
    keep[bad_row] = False
    xs, ys = (x[0][keep], y[0]) if cloud == "x" else (x[0], y[0][keep])
    with torch.no_grad():
        fx, fy = M._nn_sq_dist(x[0], y[0]), M._nn_sq_dist(y[0], x[0])
        cx, cy = M._nn_sq_dist(xs, ys), M._nn_sq_dist(ys, xs)
    if cloud == "x":                                                # the bad row is a query of fx and a reference of fy
        assert not torch.isfinite(fx[bad_row])
        assert torch.equal(fx[keep], cx) and torch.equal(fy, cy)
    else:
        assert not torch.isfinite(fy[bad_row])
        assert torch.equal(fy[keep], cy) and torch.equal(fx, cx)


# ---- dist_stats --------------------------------------------------------------------------------------------------------------
def gpu_ds(h, d, t):
    dt = torch.as_tensor(np.ascontiguousarray(d, np.float64), device=DEV)
    tt = torch.as_tensor(np.ascontiguousarray(t, np.float64), device=DEV)
    s = torch.full((1,), -7.0, dtype=torch.float64, device=DEV)
    c = torch.full((max(tt.shape[0], 1),), -7, dtype=torch.int64, device=DEV)
    h.dist_stats(dt, tt, s, c[: tt.shape[0]])
    return s.cpu().numpy(), c[: tt.shape[0]].cpu().numpy()


@pytest.mark.parametrize("n", [1, 255, 256, 257, 262_143, 262_144, 262_145, 3_000_001])
def test_dist_stats_sum_bit_exact_where_the_grid_changes(h, n):
    g = np.random.default_rng(n)
    d = np.abs(g.standard_normal(n)) * np.exp(g.uniform(-20, 20, n))     # magnitudes that make the order visible
    t = np.linspace(0.05, 0.1, 100)
    s, c = gpu_ds(h, d, t)
    assert same_bits(s, [mr.ordered_sum(d)])
    assert np.array_equal(c, mr.counts_below(d, t))


@pytest.mark.parametrize("nt", [0, 1, 100, 4096])
def test_dist_stats_thresholds_at_and_around_each_distance(h, nt):
    g = np.random.default_rng(nt + 1)
    t = np.sort(g.uniform(0.0, 0.2, nt))
    if nt > 4:
        t[nt // 2] = t[nt // 2 + 1] = t[nt // 2 + 2]                 # duplicates
    d = np.concatenate([t, np.nextafter(t, 0.0), np.nextafter(t, 1.0), g.uniform(0, 0.25, 5000), [0.0, 0.2]])
    d = d[g.permutation(d.shape[0])]
    s, c = gpu_ds(h, d, t)
    assert same_bits(s, [mr.ordered_sum(d)])
    assert c.shape == (nt,) and np.array_equal(c, [(d < x).sum() for x in t])


def test_dist_stats_refuses_4097_thresholds(h):
    with pytest.raises(RuntimeError, match="dist_stats"):
        gpu_ds(h, np.ones(10), np.linspace(0, 1, 4097))


@pytest.mark.parametrize("bad", ["nan", "inf", "both"])
def test_dist_stats_non_finite_distances_are_never_counted(h, bad):
    g = np.random.default_rng(7)
    d = g.uniform(0, 0.2, 300_000)
    vals = {"nan": [np.nan], "inf": [np.inf], "both": [np.nan, np.inf]}[bad]
    d[g.choice(d.shape[0], 50, replace=False)] = np.resize(vals, 50)
    t = np.concatenate([np.linspace(0.0, 0.2, 200), [np.inf]])
    s, c = gpu_ds(h, d, t)
    assert np.array_equal(c, [(d < x).sum() for x in t])
    assert c[-1] == int(np.isfinite(d).sum())
    assert (np.isnan(s[0]) if bad != "inf" else s[0] == np.inf) and same_bits(s, [mr.ordered_sum(d)])


@pytest.mark.parametrize("order", ["descending", "shuffled", "nan"])
def test_evaluate_scan_counts_thresholds_in_any_order(order):
    g = np.random.default_rng(13)
    gt = g.uniform(-20, 20, (60_000, 3))
    pred = gt[g.choice(gt.shape[0], 40_000, replace=False)] + g.normal(0, 0.06, (40_000, 3))
    t = np.linspace(0.1, 0.05, 100)
    t = {"descending": t, "shuffled": g.permutation(t), "nan": np.concatenate([t[:40], [np.nan], t[40:], [np.nan]])}[order]
    rec = M.evaluate_scan(gt, pred, thresholds=t, voxel_sizes=(), hist=False)
    d_pg, d_gp = M.nn_distance(pred, gt).cpu().numpy(), M.nn_distance(gt, pred).cpu().numpy()
    assert np.array_equal(rec.thresholds, t, equal_nan=True)
    assert np.array_equal(rec.cnt_pred_to_gt, [(d_pg < x).sum() for x in t])
    assert np.array_equal(rec.cnt_gt_to_pred, [(d_gp < x).sum() for x in t])
    assert rec.sum_pred_to_gt == mr.ordered_sum(d_pg) and rec.sum_gt_to_pred == mr.ordered_sum(d_gp)


# ---- Jensen-Shannon distance -------------------------------------------------------------------------------------------------
def gpu_jsd(h, a, b):
    at = torch.as_tensor(np.ascontiguousarray(a, np.uint32).view(np.int32), device=DEV)
    bt = torch.as_tensor(np.ascontiguousarray(b, np.uint32).view(np.int32), device=DEV)
    out = torch.full((1,), -7.0, dtype=torch.float64, device=DEV)
    h.jsd(at, bt, out)
    return float(out.item())


def _hists(n, seed, shared=0.7):
    g = np.random.default_rng(seed)
    a, b = g.integers(0, 50, n).astype(np.uint32), g.integers(0, 50, n).astype(np.uint32)
    a[g.random(n) > shared] = 0
    b[g.random(n) > shared] = 0
    a[0] += 1
    b[-1] += 1
    return a, b


@pytest.mark.parametrize("n", [1, 255, 256, 257, 262_144, 262_145, 200 ** 3])
def test_jsd_within_the_bound(h, n):
    a, b = _hists(n, n)
    v = gpu_jsd(h, a, b)
    assert mr.within_jsd_bound(v, a, b), (v, mr.jsd_bound(a, b))


def test_jsd_identical_disjoint_and_empty(h):
    a, _ = _hists(262_145, 1)
    assert gpu_jsd(h, a, a) == 0.0
    a = np.zeros(100_000, np.uint32)
    b = np.zeros(100_000, np.uint32)
    a[:50_000:3], b[50_000::7] = 5, 11                              # disjoint supports
    v = gpu_jsd(h, a, b)
    assert mr.within_jsd_bound(v, a, b) and abs(v - np.sqrt(np.log(2.0))) <= 1e-13
    z = np.zeros(100_000, np.uint32)
    assert np.isnan(gpu_jsd(h, a, z)) and np.isnan(gpu_jsd(h, z, b)) and np.isnan(gpu_jsd(h, z, z))


def test_jsd_counts_that_need_64_bit_totals(h):
    g = np.random.default_rng(17)
    n = 300_000
    a = np.where(g.random(n) < 0.3, np.uint32(2 ** 32 - 1), g.integers(0, 2 ** 32, n, dtype=np.uint32)).astype(np.uint32)
    b = np.where(g.random(n) < 0.5, np.uint32(2 ** 32 - 1), np.uint32(0)).astype(np.uint32)
    b[0] = 2 ** 32 - 1
    assert int(a.sum(dtype=np.uint64)) > 2 ** 40
    v = gpu_jsd(h, a, b)
    assert mr.within_jsd_bound(v, a, b), (v, mr.jsd_bound(a, b))


# ---- occupancy, confusion, BEV -------------------------------------------------------------------------------------------------
OCC_BINS = [1, 7, 31, 33, 333, 1000, 2048]


def edge_points(edges, g):
    """every edge and one ulp either side on each axis, +-50 and just outside, +-0 on the middle edge, and rows with a NaN or
    +-inf in one coordinate (dropped)"""
    e = np.asarray(edges)
    vals = np.concatenate([e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf),
                           [-0.0, 0.0, 50.0, -50.0, np.nextafter(50.0, 100.0), np.nextafter(-50.0, -100.0)]])
    parts = []
    for axis in range(3):
        p = vals[g.integers(0, vals.shape[0], (vals.shape[0], 3))]
        p[:, axis] = vals
        parts.append(p)
    mid = e[e.shape[0] // 2]
    parts.append(np.array([[-0.0, 0.0, 0.0], [0.0, -0.0, -0.0], [-0.0, -0.0, -0.0], [mid, -mid, mid], [-mid, mid, -mid]]))
    parts.append(_nonfinite_rows(g, 60) * 0.1)
    p = np.concatenate(parts)
    return p[g.permutation(p.shape[0])]


def gpu_occupancy(h, pts, edges, counts):
    bins = edges.shape[0] - 1
    t = torch.as_tensor(np.ascontiguousarray(pts), device=DEV)
    e = torch.as_tensor(edges, device=DEV)
    bits = torch.empty((bins ** 3 + 31) // 32, dtype=torch.int32, device=DEV)
    cnt = torch.empty(bins ** 3, dtype=torch.int32, device=DEV) if counts else None
    n_in = torch.full((1,), -7, dtype=torch.int64, device=DEV)
    h.voxel_occupancy(t, e, bits, cnt, n_in)
    return bits, cnt, int(n_in.item())


def set_cells(bits):
    """the set bits' cell numbers (int64, ascending), decoded on the device from the nonzero words"""
    nz = torch.nonzero(bits).squeeze(1)
    w = bits[nz]
    sh = torch.arange(32, device=bits.device, dtype=torch.int32)
    m = ((w[:, None] >> sh) & 1).bool()
    return torch.sort((nz[:, None] * 32 + sh.long())[m]).values.cpu().numpy()


@pytest.mark.parametrize("bins", OCC_BINS)
def test_occupancy_confusion_and_bev_against_sparse_cells(h, bins):
    g = np.random.default_rng(bins)
    edges = np.linspace(-50, 50, bins + 1)
    gt = edge_points(edges, g)
    pred = np.concatenate([gt[g.permutation(gt.shape[0])[: gt.shape[0] // 2]], edge_points(edges, g)[: gt.shape[0] // 3]])
    want_gt, want_n, want_in = mr.occupancy(gt, edges)
    want_pred, _, want_in_pred = mr.occupancy(pred, edges)
    counts = bins <= 333
    bits_gt, cnt, n_in = gpu_occupancy(h, gt, edges, counts)
    assert n_in == want_in
    assert np.array_equal(set_cells(bits_gt), want_gt)
    if bins == 2048:
        assert want_gt.max() >= 2 ** 32                             # the case reaches past cell 2^32
    if counts:
        c = cnt.cpu().numpy().view(np.uint32)
        assert np.array_equal(np.nonzero(c)[0], want_gt) and np.array_equal(c[want_gt], want_n)
    del cnt
    bits_pred, _, n_in_pred = gpu_occupancy(h, pred, edges, False)
    assert n_in_pred == want_in_pred and np.array_equal(set_cells(bits_pred), want_pred)
    out = torch.full((3,), -7, dtype=torch.int64, device=DEV)
    h.occupancy_confusion(bits_gt, bits_pred, bins ** 3, out)
    assert tuple(out.cpu().tolist()) == mr.confusion(want_gt, want_pred)
    bev = torch.full((bins * bins,), -7, dtype=torch.int32, device=DEV)
    h.occupancy_bev(bits_gt, bins, bev)
    bev = bev.cpu().numpy()
    col, n = mr.bev(want_gt, bins)
    assert np.array_equal(np.nonzero(bev)[0], col) and np.array_equal(bev[col], n)
