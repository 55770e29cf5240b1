"""The exact self-k-NN (lb2_pc_knn) and the point normals (lb2_pc_normals) at their edges, against tests/knn_reference.py and
tests/normals_oracle.py:
  * k-NN rows and d² bit for bit against the fp64 brute force for k in {1, 2, 8, 27, 30, 31, 32}: lattices whose k-th slot ties
    across leaves and outside the seed window, fp32 node boxes that are coarse or leave the fp32 range, d² that overflow or
    underflow, signed zeros, duplicate groups longer than the seed window, tree sizes at the leaf-doubling edge (up to 2²⁰ + 1),
    fewer finite points than k and none;
  * normals of tilted planes and lines, isotropic lattice interiors and k = 1, 2 (bit for bit), clouds offset by 1e6 / 1e8 where
    the one-pass covariance cancels, and coordinates where it overflows;
  * rows with a NaN or infinite coordinate leave the tree's root box and the finite rows' order alone and sort last — checked on
    the tree's bytes before any search runs, so a regression fails at once instead of walking every leaf for every point — and
    then k-NN, normals and nearest-neighbour distances equal those of the finite rows alone, bit for bit."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import knn_reference as R
import normals_oracle as O
from lidiff_b200 import metrics as M
from lidiff_b200 import normals as N

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KS = (1, 2, 8, 27, 30, 31, 32)
_REF = {}


@pytest.fixture(scope="module")
def h():
    from lidiff_b200 import _lib
    return _lib.get_handle(DEV)


def gpu_knn(p, k):
    idx, d2 = N.knn(np.ascontiguousarray(p, np.float64), k, device=DEV)
    return idx.cpu().numpy().astype(np.int64), d2.cpu().numpy()


def assert_rows(idx, d2, want_i, want_d, what=""):
    assert idx.shape == want_i.shape, (what, idx.shape, want_i.shape)
    bad = np.nonzero((idx != want_i).any(1) | (d2.view(np.int64) != want_d.view(np.int64)).any(1))[0]
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} rows differ, first {bad[:3]}: gpu {idx[bad[:1]]} {d2[bad[:1]]}, " \
                              f"want {want_i[bad[:1]]} {want_d[bad[:1]]}"


def reference32(name, p):
    """the brute force at k = 32, once per cloud: its k-prefix is the k-NN for every smaller k ((d², index) is a total order)"""
    if name not in _REF:
        _REF[name] = R.knn(p, 32)
    return _REF[name]


def assert_no_repeats(idx):
    s = np.sort(idx, 1)
    assert not ((s[:, 1:] == s[:, :-1]) & (s[:, 1:] >= 0)).any()


# ---- k-NN ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", sorted(set(R.KNN_CLOUDS) - {"identical_20000"}))
def test_knn_bit_exact_on_edge_clouds(name, k):
    p = R.cloud(name)
    wi, wd = reference32(name, p)
    ke = min(k, p.shape[0])
    idx, d2 = gpu_knn(p, k)
    assert_rows(idx, d2, wi[:, :ke], wd[:, :ke], name)
    assert_no_repeats(idx)
    if name == "subnormal":                                         # every d² is 0: the k lowest indices, itself possibly absent
        assert (d2 == 0).all() and (idx == np.arange(k)).all()
    if name == "overflow_1e200":                                    # only the point and an exact copy have a finite d²
        assert (idx[:, 0] >= 0).all() and (idx[:, 2:] == -1).all() and np.isinf(d2[:, 2:]).all() and (d2[idx >= 0] == 0).all()
    if name.startswith("dup"):                                      # the lowest indices of the group, none twice
        grp = np.unique(p, axis=0, return_inverse=True)[1].reshape(-1)
        first = {gid: np.flatnonzero(grp == gid)[:k] for gid in np.unique(grp)}
        assert all(np.array_equal(idx[i], first[grp[i]]) for i in range(0, p.shape[0], 7))


@pytest.mark.parametrize("k", [1, 8, 32])
def test_knn_20000_identical_points(k):
    idx, d2 = gpu_knn(R.cloud("identical_20000"), k)
    assert (idx == np.arange(k)).all() and (d2 == 0).all()


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 31, 32, 33, 65])
def test_knn_tree_shape_sizes(n):
    p = np.random.default_rng(n).normal(0, 3, (n, 3))
    wi, wd = R.knn(p, 32)
    for k in KS:
        idx, d2 = gpu_knn(p, k)
        assert_rows(idx, d2, wi[:, :min(k, n)], wd[:, :min(k, n)], f"n={n} k={k}")


@pytest.mark.parametrize("n", [1_048_576, 1_048_577])
def test_knn_leaf_doubling_edge(n):
    """2^17 full leaves, and one point more (twice the leaves, most of them empty): 1 000 sampled rows and the last 5 against the
    brute force for every k, every row's d² against cKDTree's distances at k = 32"""
    g = np.random.default_rng(n)
    p = g.normal(0, 20, (n, 3))
    rows = np.concatenate([g.choice(n - 5, 1000, replace=False), np.arange(n - 5, n)])
    wi, wd = R.knn(p, 32, rows)
    for k in KS:
        idx, d2 = gpu_knn(p, k)
        assert_rows(idx[rows], d2[rows], wi[:, :k], wd[:, :k], f"k={k}")
    kd, _ = cKDTree(p).query(p, k=32, workers=-1)
    assert np.abs(np.sqrt(d2) - kd).max() <= 1e-12 * max(1.0, kd.max())


def test_knn_fewer_finite_points_than_k_and_none():
    g = np.random.default_rng(11)
    p = np.concatenate([g.uniform(-1, 1, (20, 3)), [[np.nan, 0, 0], [0, np.inf, 0], [-np.inf] * 3]])
    p = p[g.permutation(p.shape[0])]
    for k in (27, 32):
        idx, d2 = gpu_knn(p, k)
        assert_rows(idx, d2, *R.knn(p, k), f"k={k}")
        assert ((idx >= 0).sum(1) == np.where(np.isfinite(p).all(1), 20, 0)).all()
    for bad in (np.full((40, 3), np.nan), np.full((9, 3), -np.inf), np.array([[np.nan, 1.0, 2.0]])):
        idx, d2 = gpu_knn(bad, 8)
        assert (idx == -1).all() and np.isinf(d2).all()


# ---- normals -----------------------------------------------------------------------------------------------------------------
def check_normals(p, nrm, k=30):
    """the existing rule: 1 - |n·n_ref| <= 1e-9 where the eigen-gap is >= 1e-6, the same sign where every sign decision has a
    margin; and bit for bit where the solver takes no trigonometric branch (the covariance is bit-exact, only acos / cos differ)"""
    idx, _ = R.knn(p, k)
    want, diag, cov = O.normals_from_idx(p, idx)
    with np.errstate(invalid="ignore"):
        gap = np.isfinite(cov).all((1, 2)) & (O.eigen_gap(np.nan_to_num(cov)) >= 1e-6)
    dots = (nrm * want).sum(1)
    assert (1 - np.abs(dots[gap])).max(initial=0.0) <= 1e-9
    clear = O.clear_sign(diag) & gap
    assert (dots[clear] > 0).all(), f"{(dots[clear] <= 0).sum()} clear points with the other sign"
    no_trig = diag["half_det"] == 0
    assert np.array_equal(nrm[no_trig].view(np.int64), want[no_trig].view(np.int64))
    return want, gap, cov


def _rotation(g):
    q, r = np.linalg.qr(g.normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


def test_normals_of_tilted_planes_and_lines():
    g = np.random.default_rng(12)
    rot = _rotation(g)
    plane = np.c_[g.uniform(-2, 2, (4000, 2)), np.zeros(4000)] @ rot.T + [3.0, -1.0, 0.5]
    nrm = N.estimate_normals(plane, device=DEV).cpu().numpy()
    _, gap, _ = check_normals(plane, nrm)
    assert gap.mean() > 0.95 and np.abs(np.abs(nrm @ rot[:, 2]) - 1).max() <= 1e-9
    for d in (rot[:, 0], np.array([1.0, 1.0, 1.0]) / np.sqrt(3.0)):
        line = g.uniform(-5, 5, (1500, 1)) * d + [1.0, 2.0, -3.0]
        nrm = N.estimate_normals(line, device=DEV).cpu().numpy()
        check_normals(line, nrm)
        assert np.abs(nrm @ d).max() <= 1e-6 and np.abs(np.linalg.norm(nrm, axis=1) - 1).max() <= 1e-12


def test_normals_of_isotropic_lattice_interiors_bit_exact():
    """k = 27 on Z³: an interior point's neighbours are its 3×3×3 cube, whose covariance is (2/3) I up to the rounding of each
    diagonal entry; the off-diagonal entries are exactly 0, so the solver picks an axis without trigonometry"""
    p = R.cloud("z3")
    nrm = N.estimate_normals(p, knn=27, device=DEV).cpu().numpy()
    idx, _ = R.knn(p, 27)
    want, diag, cov = O.normals_from_idx(p, idx)
    lo, hi = p.min(0), p.max(0)
    interior = ((p > lo) & (p < hi)).all(1)
    assert interior.sum() == 12 ** 3
    off = cov[interior][:, [0, 0, 1], [1, 2, 2]]
    assert (off == 0).all() and (np.abs(np.diagonal(cov[interior], axis1=1, axis2=2) - 2 / 3) <= 1e-13).all()
    assert np.unique(want[interior], axis=0).shape[0] == 3          # the rounding of each diagonal entry picks the axis
    assert np.array_equal(nrm[interior].view(np.int64), want[interior].view(np.int64))
    check_normals(p, nrm, 27)


@pytest.mark.parametrize("k", [1, 2])
def test_normals_below_three_neighbours_are_z(k):
    p = np.random.default_rng(k).normal(0, 4, (3000, 3))
    nrm = N.estimate_normals(p, knn=k, device=DEV).cpu().numpy()
    assert np.array_equal(nrm, np.tile([0.0, 0.0, 1.0], (3000, 1)))
    assert np.array_equal(nrm, O.normals_from_idx(p, R.knn(p, k)[0])[0])


@pytest.mark.parametrize("offset", [1e6, 1e8])
def test_normals_of_offset_clouds_where_the_covariance_cancels(offset):
    """open3d's one-pass covariance E[ppᵀ] − E[p]E[p]ᵀ loses most of its digits at these offsets; the kernel computes the same
    cancelled covariance bit for bit, so it still meets the rule against the restatement"""
    g = np.random.default_rng(int(np.log10(offset)))
    rot = _rotation(g)
    patch = np.c_[g.uniform(-1, 1, (3000, 2)), g.normal(0, 0.01, 3000)] @ rot.T
    p = patch + np.array([1.0, -0.5, 0.25]) * offset
    nrm = N.estimate_normals(p, device=DEV).cpu().numpy()
    want, gap, _ = check_normals(p, nrm)
    assert gap.any()


@pytest.mark.parametrize("offset", [1e154, 1e155, 1e160])
def test_normals_where_the_covariance_overflows(offset):
    """a tilted slab of extent 1e150 (its squared distances are finite) around a point at `offset`, where the cumulants x·x
    overflow: a NaN or infinite covariance entry gives (0, 0, 1) in the kernel and in the restatement"""
    g = np.random.default_rng(int(np.log10(offset)))
    p = (g.normal(0, 1, (3000, 3)) * [1.0, 1.0, 1e-3]) @ _rotation(g).T * 1e150 + np.array([0.6, -0.8, 0.5]) * offset
    nrm = N.estimate_normals(p, device=DEV).cpu().numpy()
    want, _, cov = check_normals(p, nrm)
    bad = ~np.isfinite(cov).all((1, 2))
    assert bad.mean() > 0.5 and (nrm[bad] == [0.0, 0.0, 1.0]).all() and not np.isnan(nrm).any()
    assert np.array_equal(nrm[bad], want[bad])


# ---- non-finite rows and the tree's shape -------------------------------------------------------------------------------------
def tree_view(tree):
    """the tree's bytes (csrc/metrics.cu): header (6 order-preserving uint64 bounding-box keys, nleaf and n as int32 at byte 48),
    nodes float[2 nleaf][8] {lo xyz, 0, hi xyz, 0} (root at node 1), sorted points double4 (x, y, z, original index)"""
    b = tree.cpu().numpy()
    nleaf, n = (int(v) for v in b[48:56].view(np.int32))
    nodes = b[64:64 + 2 * nleaf * 32].view(np.float32).reshape(2 * nleaf, 8)
    sp = b[64 + 2 * nleaf * 32:64 + 2 * nleaf * 32 + nleaf * 8 * 32].view(np.float64).reshape(-1, 4)
    return {"nleaf": nleaf, "n": n, "bbox": R.unkey(b[:48].view(np.uint64)), "root": nodes[1],
            "order": sp[:n, 3].astype(np.int64)}


@pytest.fixture(scope="module")
def refined():
    return O.refined_like()


BAD_ROWS = {"inf": [np.inf, 0.0, 0.0], "-inf": [0.0, 1.0, -np.inf], "nan_row": [np.nan] * 3,
            "signed_nan": [0.0, np.copysign(np.nan, -1.0), 2.0]}


@pytest.mark.parametrize("bad", list(BAD_ROWS) + ["all"])
def test_non_finite_rows_do_not_shape_the_tree(h, refined, bad):
    g = np.random.default_rng(len(bad))
    rows = np.array(list(BAD_ROWS.values()) if bad == "all" else [BAD_ROWS[bad]] * 3)
    pos = np.sort(g.choice(refined.shape[0] + rows.shape[0], rows.shape[0], replace=False))
    is_bad = np.zeros(refined.shape[0] + rows.shape[0], bool)
    is_bad[pos] = True
    p = np.empty((is_bad.shape[0], 3))
    p[is_bad], p[~is_bad] = rows, refined
    keep = np.flatnonzero(~is_bad)                                  # finite-cloud index -> mixed-cloud index
    pt, ft = torch.as_tensor(p, device=DEV), torch.as_tensor(refined, device=DEV)
    mixed, fin = tree_view(h.pc_tree(pt)), tree_view(h.pc_tree(ft))
    # structure first: a tree shaped by a non-finite row would make every search below visit every leaf
    assert mixed["nleaf"] == fin["nleaf"] and mixed["n"] == p.shape[0]
    assert np.array_equal(mixed["root"], fin["root"]), f"root box {mixed['root']} != finite rows' {fin['root']}"
    assert np.array_equal(mixed["bbox"], fin["bbox"])
    order = mixed["order"]
    assert not is_bad[order[:refined.shape[0]]].any(), "a non-finite row sorts before a finite one"
    assert np.array_equal(order[:refined.shape[0]], keep[fin["order"]]), "the finite rows' order changed"
    assert np.array_equal(order, R.tree_layout(p)["order"])
    # then the searches: the finite rows' results in the original indices, bit for bit
    for k in (30,):
        idx, d2 = (t.cpu().numpy() for t in N.knn(pt, k, device=DEV))
        fi, fd = (t.cpu().numpy() for t in N.knn(ft, k, device=DEV))
        assert (idx[is_bad] == -1).all() and np.isinf(d2[is_bad]).all()
        assert np.array_equal(idx[~is_bad], keep[fi]) and np.array_equal(d2[~is_bad].view(np.int64), fd.view(np.int64))
    nrm, fnrm = N.estimate_normals(pt, device=DEV).cpu().numpy(), N.estimate_normals(ft, device=DEV).cpu().numpy()
    assert np.isnan(nrm[is_bad]).all() and np.array_equal(nrm[~is_bad].view(np.int64), fnrm.view(np.int64))
    q = np.concatenate([refined[g.choice(refined.shape[0], 20_000, replace=False)] + g.normal(0, 0.05, (20_000, 3)), rows])
    d, j = (t.cpu().numpy() for t in M.nn_distance(q, pt, return_index=True, device=DEV))
    fd, fj = (t.cpu().numpy() for t in M.nn_distance(q, ft, return_index=True, device=DEV))
    assert np.array_equal(d.view(np.int64), fd.view(np.int64)) and np.array_equal(j[:20_000], keep[fj[:20_000]])
    assert (j[20_000:] == -1).all() and (fj[20_000:] == -1).all()
    d, fd = M.nn_distance(pt, ft, device=DEV).cpu().numpy(), M.nn_distance(ft, ft, device=DEV).cpu().numpy()
    assert np.isinf(d[is_bad]).all() and np.array_equal(d[~is_bad].view(np.int64), fd.view(np.int64))
