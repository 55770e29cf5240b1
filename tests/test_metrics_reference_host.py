"""The restatements of tests/metrics_reference.py on the CPU: they agree with scipy's cKDTree, jensenshannon and np.histogramdd on
small hand-checkable inputs; the JSD bound admits a 1-ulp log and rejects logf, a dropped block partial and a dropped q term; the
ordered sum is not a reordering in disguise; the fake backends follow lb2_pc_nn's -1 contract; and evaluate_scan counts any
threshold order as numpy does."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree
from scipy.spatial.distance import jensenshannon

import metrics_reference as mr

SIZES = [1, 255, 256, 257, 262_143, 262_144, 262_145, 3_000_001]


# ---- nearest neighbour -------------------------------------------------------------------------------------------------------
def test_nn_agrees_with_ckdtree_and_takes_the_lowest_index():
    g = np.random.default_rng(0)
    r = g.uniform(-3, 3, (400, 3))
    r = np.concatenate([r, r[:50], r[::-1]])                        # duplicates: the first copy must win
    q = np.concatenate([g.uniform(-4, 4, (300, 3)), r[:20]])
    d, j = mr.nn(q, r)
    kd, kj = cKDTree(r).query(q)
    assert np.abs(d - kd).max() <= 1e-12
    assert np.array_equal(j[300:], np.arange(20))
    first = {tuple(p): i for i, p in reversed(list(enumerate(r)))}
    assert np.array_equal(j[:300], [first[tuple(r[k])] for k in kj[:300]])


def test_nn_lattice_ties_and_signed_zero():
    ax = np.arange(3, dtype=np.float64)
    lat = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    d, j = mr.nn(np.array([[0.5, 0.5, 0.5]]), lat)                  # 8 lattice points at the same distance
    assert j[0] == 0 and d[0] == np.sqrt(0.75)
    r = np.array([[-0.0, 0.0, 0.0], [0.0, -0.0, 0.0]])
    d, j = mr.nn(np.array([[0.0, 0.0, 0.0], [-0.0, -0.0, -0.0]]), r[::-1])
    assert np.array_equal(j, [0, 0]) and np.array_equal(d, [0.0, 0.0])


def test_nn_non_finite_contract():
    r = np.array([[np.nan, 0, 0], [1.0, 1.0, 1.0], [np.inf, 0, 0], [0.0, 0.0, 0.0]])
    q = np.array([[0.1, 0, 0], [np.nan, 0, 0], [0, -np.inf, 0], [1e200, 0, 0], [1e150, 0, 0], [np.nan] * 3])
    d, j = mr.nn(q, r)
    assert np.array_equal(j, [3, -1, -1, -1, 1, -1])               # at 1e150 the points 1 and 3 tie in fp64
    assert d[0] == 0.1 and d[4] == np.sqrt(1e150 * 1e150) and np.isinf(d[[1, 2, 3, 5]]).all()
    d, j = mr.nn(q[:1], np.array([[np.nan, 0, 0], [0, np.inf, 0]]))
    assert j[0] == -1 and d[0] == np.inf


# ---- dist_stats --------------------------------------------------------------------------------------------------------------
def test_ordered_sum_small_cases_are_exact():
    assert mr.ordered_sum([1.5]) == 1.5
    v = np.arange(1000, dtype=np.float64)                           # every partial sum is an exact integer
    assert mr.ordered_sum(v) == v.sum()
    assert np.isnan(mr.ordered_sum([1.0, np.nan, 2.0])) and mr.ordered_sum([1.0, np.inf]) == np.inf


@pytest.mark.parametrize("n", SIZES)
def test_ordered_sum_is_near_the_exact_sum(n):
    v = np.random.default_rng(n).exponential(1.0, n)
    exact = float(np.sum(v.astype(np.longdouble)))
    assert abs(mr.ordered_sum(v) - exact) <= 2 * mr.U * mr.path_adds(n) * exact


def test_ordered_sum_is_not_a_reordering():
    """the restatement differs from a reversed block order and from numpy's pairwise order on some tested n, so matching it bit
    for bit pins the kernel's order"""
    diff_rev, diff_np = [], []
    for n in SIZES:
        v = np.random.default_rng(n + 1).standard_normal(n) * np.exp(np.random.default_rng(n + 2).uniform(-20, 20, n))
        s = mr.ordered_sum(v)
        diff_rev.append(s != mr.ordered_sum(v, reverse_blocks=True))
        diff_np.append(s != float(np.sum(v)))
    assert any(diff_rev) and any(diff_np)


def test_counts_equal_numpy_per_threshold():
    d = np.array([0.0, 0.05, 0.1, np.nextafter(0.1, 1), np.nextafter(0.1, 0), np.inf, np.nan, 0.2])
    t = np.array([0.1, 0.05, np.nan, 0.1, -np.inf, np.inf, 0.0, np.nextafter(0.1, 1)])
    want = np.array([(d < x).sum() for x in t])
    assert np.array_equal(mr.counts_below(d, t), want)


def test_kernel_search_equals_numpy_only_for_ascending_thresholds():
    g = np.random.default_rng(3)
    d = g.uniform(0, 0.2, 5000)
    t = np.linspace(0.05, 0.1, 100)
    assert np.array_equal(mr.ds_kernel_counts(d, t), mr.counts_below(d, t))
    tt = np.concatenate([t[:50], t[:50]])                           # duplicates still ascending
    assert np.array_equal(mr.ds_kernel_counts(d, np.sort(tt)), mr.counts_below(d, np.sort(tt)))
    for bad in (t[::-1], g.permutation(t), np.concatenate([t[:10], [np.nan], t[10:]])):
        assert not np.array_equal(mr.ds_kernel_counts(d, bad), mr.counts_below(d, bad))


# ---- Jensen-Shannon distance -------------------------------------------------------------------------------------------------
def _hists(n, seed, shared=0.7):
    g = np.random.default_rng(seed)
    a = g.integers(0, 50, n).astype(np.uint32)
    b = g.integers(0, 50, n).astype(np.uint32)
    a[g.random(n) > shared] = 0
    b[g.random(n) > shared] = 0
    if a.sum() == 0:
        a[0] = 3
    if b.sum() == 0:
        b[-1] = 2
    return a, b


def test_jsd_agrees_with_scipy_and_hand_values():
    a, b = _hists(1000, 0)
    want = jensenshannon(a / a.sum(), b / b.sum())
    assert mr.jsd(a, b) == pytest.approx(want, rel=1e-13)
    assert mr.within_jsd_bound(want, a, b)
    x = np.array([3, 0, 5], np.uint32)
    assert mr.jsd(x, x) == 0.0
    assert mr.jsd(np.array([1, 0], np.uint32), np.array([0, 1], np.uint32)) == pytest.approx(np.sqrt(np.log(2)), rel=1e-15)
    assert np.isnan(mr.jsd(x, np.zeros(3, np.uint32))) and np.isnan(mr.jsd(np.zeros(3, np.uint32), np.zeros(3, np.uint32)))
    assert mr.within_jsd_bound(float("nan"), x, np.zeros(3, np.uint32)) and not mr.within_jsd_bound(0.5, x, np.zeros(3, np.uint32))


def _ulp_log(seed):
    g = np.random.default_rng(seed)

    def log(x):
        y = np.log(x)
        s = g.integers(-1, 2, y.shape)
        return np.where(s > 0, np.nextafter(y, np.inf), np.where(s < 0, np.nextafter(y, -np.inf), y))
    return log


def _logf(x):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log(x.astype(np.float32)).astype(np.float64)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 262_144, 262_145])
def test_jsd_bound_admits_a_1_ulp_log(n):
    a, b = _hists(n, n)
    for seed in range(3):
        assert mr.within_jsd_bound(mr.jsd(a, b, log=_ulp_log(seed)), a, b)


@pytest.mark.parametrize("n", [256, 257, 262_144, 262_145])
def test_jsd_bound_rejects_logf_a_dropped_block_and_a_dropped_q_term(n):
    a, b = _hists(n, n + 7)
    assert not mr.within_jsd_bound(mr.jsd(a, b, log=_logf), a, b)
    assert not mr.within_jsd_bound(mr.jsd(a, b, drop_shared_q=True), a, b)
    nblk = mr.rd_blocks(n)
    if nblk > 1:
        assert not mr.within_jsd_bound(mr.jsd(a, b, drop_block=nblk // 2), a, b)


def test_jsd_bound_holds_for_64_bit_totals():
    a = np.full(4, 2 ** 32 - 1, np.uint32)
    b = np.array([2 ** 32 - 1, 1, 2 ** 32 - 1, 0], np.uint32)
    p = a / (4.0 * (2 ** 32 - 1))
    bb = b.astype(np.float64) / float(b.sum(dtype=np.uint64))
    assert mr.within_jsd_bound(jensenshannon(p, bb), a, b)


# ---- occupancy -----------------------------------------------------------------------------------------------------------------
def test_occupancy_agrees_with_histogramdd():
    e = np.linspace(-50, 50, 8)
    g = np.random.default_rng(5)
    pts = np.concatenate([e[g.integers(0, 8, (500, 3))], g.uniform(-60, 60, (500, 3)),
                          [[50.0, 50.0, 50.0], [-50.0, 0.0, np.nextafter(50.0, 100)], [np.nan, 0, 0], [0, np.inf, 0], [-0.0, 0.0, -0.0]]])
    h = np.histogramdd(pts[np.isfinite(pts).all(1)], bins=7, range=[[-50, 50]] * 3)[0].reshape(-1)
    c, n, n_in = mr.occupancy(pts, e)
    assert np.array_equal(c, np.nonzero(h)[0]) and np.array_equal(n, h[h > 0]) and n_in == int(h.sum())
    col, cnt = mr.bev(c, 7)
    hb = (h.reshape(7, 7, 7) > 0).sum(-1).reshape(-1)
    assert np.array_equal(col, np.nonzero(hb)[0]) and np.array_equal(cnt, hb[hb > 0])
    c2, _, _ = mr.occupancy(pts[::2] + 1.0, e)
    a, b = h > 0, np.isin(np.arange(343), c2)
    assert mr.confusion(c, c2) == ((a & b).sum(), (a & ~b).sum(), (~a & b).sum())


def test_occupancy_cells_past_2_to_the_32():
    e = np.linspace(-50, 50, 2049)
    c = mr.cells(np.array([[50.0, 50.0, 50.0], [e[1024], -50.0, -50.0]]), e)
    assert c.dtype == np.int64 and list(c) == [2048 ** 3 - 1, 1024 * 2048 * 2048]


# ---- the fake backends follow the kernels' contracts ---------------------------------------------------------------------------
def _fake_nn(handle, q, r):
    qt, rt = torch.as_tensor(q), torch.as_tensor(r)
    dist = torch.empty(q.shape[0], dtype=torch.float64)
    idx = torch.empty(q.shape[0], dtype=torch.int32)
    handle.pc_nn(qt, handle.pc_tree(rt), dist, idx)
    return dist.numpy(), idx.numpy()


@pytest.mark.parametrize("backend", ["metrics", "refine"])
def test_fake_pc_nn_follows_the_minus_one_contract(backend):
    import fake_metrics_backend
    import fake_refine_backend
    handle = {"metrics": fake_metrics_backend.FakeMetricsHandle, "refine": fake_refine_backend.FakeRefineHandle}[backend]()
    g = np.random.default_rng(9)
    r = np.concatenate([g.uniform(-5, 5, (200, 3)), [[np.nan, 0, 0], [0, np.inf, 0]]])[::-1].copy()
    q = np.concatenate([g.uniform(-6, 6, (50, 3)), [[np.nan, 1, 1], [1, 1, -np.inf], [1e200, 0, 0]]])
    d, j = _fake_nn(handle, q, r)
    wd, wj = mr.nn(q, r)
    assert np.array_equal(j, wj) and np.array_equal(np.isinf(d), np.isinf(wd))
    fin = np.isfinite(wd)
    assert np.abs(d[fin] - wd[fin]).max() <= 1e-12                  # cKDTree's distances are not in the kernel's order
    d, j = _fake_nn(handle, q[:5], np.array([[np.nan, 0, 0], [np.inf, 1, 1]]))
    assert (j == -1).all() and np.isinf(d).all()


@pytest.mark.parametrize("order", ["descending", "shuffled", "nan"])
def test_evaluate_scan_counts_any_threshold_order(monkeypatch, order):
    import fake_metrics_backend
    from lidiff_b200 import metrics as M
    fake_metrics_backend.install(monkeypatch)
    g = np.random.default_rng(11)
    gt = g.uniform(-10, 10, (3000, 3))
    pred = gt[:2000] + g.normal(0, 0.06, (2000, 3))
    t = np.linspace(0.1, 0.05, 100)
    t = {"descending": t, "shuffled": g.permutation(t), "nan": np.concatenate([t[:30], [np.nan], t[30:], [np.nan]])}[order]
    rec = M.evaluate_scan(gt, pred, thresholds=t, voxel_sizes=(), hist=False)
    d_pg, d_gp = cKDTree(gt).query(pred)[0], cKDTree(pred).query(gt)[0]
    assert np.array_equal(rec.thresholds, t, equal_nan=True)
    assert np.array_equal(rec.cnt_pred_to_gt, [(d_pg < x).sum() for x in t])
    assert np.array_equal(rec.cnt_gt_to_pred, [(d_gp < x).sum() for x in t])
