"""The k-NN brute force and the tree-layout emulation of tests/knn_reference.py on the CPU: the brute force agrees with the normals
restatement's cKDTree-based search on ordinary clouds and with a per-row pure-Python loop on every edge cloud; the lattice and
duplicate clouds of tests/test_gpu_knn_normals_edges.py really put points tying with the k-th neighbour in other leaves than the
query's and outside the 32 sorted points that seed k_pc_knn (so those GPU tests cannot pass without the index rule deciding across
boxes); and the emulated build shows how one non-finite row collapsed the Morton grid before such rows were kept out of the tree."""
import math

import numpy as np
import pytest

import knn_reference as R
import normals_oracle as O

KS = (1, 2, 8, 27, 30, 31, 32)


def _loop_knn(p, k, rows):
    """the contract row by row in Python floats: finite d² only, (d², index) order, (-1, +inf) padding"""
    n = p.shape[0]
    ke = min(k, n)
    pts = [tuple(float(v) for v in row) for row in p]
    out_i, out_d = [], []
    for r in rows:
        qx, qy, qz = pts[r]
        cand = []
        if all(math.isfinite(v) for v in pts[r]):
            for j, (x, y, z) in enumerate(pts):
                dx, dy, dz = qx - x, qy - y, qz - z
                try:
                    d = (dx * dx + dy * dy) + dz * dz
                except OverflowError:                               # Python raises where numpy gives inf
                    continue
                if d < math.inf:
                    cand.append((d, j))
        cand.sort()
        cand = cand[:ke] + [(math.inf, -1)] * (ke - len(cand[:ke]))
        out_i.append([j for _, j in cand])
        out_d.append([d for d, _ in cand])
    return np.array(out_i, np.int64).reshape(-1, ke), np.array(out_d).reshape(-1, ke)


def _with_non_finite(p, g):
    bad = np.array([[np.inf, 0.0, 0.0], [0.0, -np.inf, 1.0], [np.nan] * 3, [1.0, 2.0, -np.nan]])
    q = np.concatenate([p, bad])
    return q[g.permutation(q.shape[0])]


def test_brute_force_agrees_with_the_normals_restatement():
    g = np.random.default_rng(0)
    for p in (g.uniform(-10, 10, (3000, 3)), g.uniform(-10, 10, (3000, 3)) * [1.0, 1.0, 0.001],
              np.repeat(g.uniform(-5, 5, (75, 3)), 40, 0)[g.permutation(3000)], g.uniform(-1, 1, (20, 3))):
        for k in (1, 8, 30, 32):
            i, d = R.knn(p, k)
            wi, wd = O.knn(p, k)
            assert np.array_equal(i, wi) and np.array_equal(d.view(np.int64), wd.view(np.int64))


@pytest.mark.parametrize("name", sorted(set(R.KNN_CLOUDS) - {"identical_20000"}) + ["non_finite"])
def test_brute_force_agrees_with_a_per_row_loop(name):
    g = np.random.default_rng(1)
    p = _with_non_finite(R.cloud("dup50"), g) if name == "non_finite" else R.cloud(name)
    rows = np.concatenate([g.choice(p.shape[0], 40, replace=False), np.flatnonzero(~np.isfinite(p).all(1))])
    i, d = R.knn(p, 32, rows)
    li, ld = _loop_knn(p, 32, rows)
    assert np.array_equal(i, li) and np.array_equal(d.view(np.int64), ld.view(np.int64))
    for k in KS:                                                    # a k-prefix is the k-NN: the (d², index) order is total
        ik, dk = R.knn(p, k, rows[:10])
        assert np.array_equal(ik, i[:10, :k]) and np.array_equal(dk, d[:10, :k])


def test_brute_force_edge_contract():
    few = np.concatenate([np.random.default_rng(2).uniform(-1, 1, (5, 3)), np.full((3, 3), np.nan)])
    i, d = R.knn(few, 8)
    assert (i[:5, :5] >= 0).all() and (i[:5, 5:] == -1).all() and np.isinf(d[:5, 5:]).all() and (i[5:] == -1).all()
    i, d = R.knn(np.full((4, 3), np.inf), 3)
    assert (i == -1).all() and np.isinf(d).all()
    i, d = R.knn(R.cloud("overflow_1e200"), 32)
    assert (i[:, 0] >= 0).all() and (i[:, 2:] == -1).all() and (i[:, 1] >= 0).sum() == 40      # only the point and an exact copy


@pytest.mark.parametrize("name", R.TIE_CLOUDS)
def test_tie_clouds_reach_past_the_leaf_and_the_seed_window(name):
    """for each k, most sampled rows have several points at exactly the k-th d² and at least one of them lies in another leaf
    than the query's and outside its seed window (k = 1 on a lattice has no tie: the point itself is alone at d² = 0)"""
    p = R.cloud(name)
    lay = R.tree_layout(p)
    rows = np.random.default_rng(3).choice(p.shape[0], 100, replace=False)
    for k in KS:
        if k == 1 and name in ("z3", "dyadic"):
            continue
        tied, out = R.ties_outside(p, k, rows, lay)
        assert ((tied >= 2) & (out >= 1)).mean() >= 0.8, (k, tied, out)


def test_duplicate_groups_are_longer_than_the_seed_window():
    for name, size in (("dup50", 50), ("dup200", 200), ("identical_20000", 20_000)):
        p = R.cloud(name)
        lay = R.tree_layout(p)
        first = np.unique(p, axis=0, return_inverse=True)[1].reshape(-1)
        for grp in np.unique(first)[:5]:
            slots = np.flatnonzero(first[lay["order"]] == grp)          # a group's copies lie in consecutive sorted slots
            assert slots.shape[0] == size and (np.diff(slots) == 1).all() and size > R.SEED


def test_emulated_codes_and_box_of_a_plain_cloud():
    p = np.random.default_rng(4).normal(0, 5, (5000, 3))
    lay = R.tree_layout(p)
    assert np.array_equal(lay["lo"], p.min(0)) and np.array_equal(lay["hi"], p.max(0))
    assert lay["codes"].max() < 2 ** 30 and np.unique(lay["codes"]).shape[0] > 4000
    assert (np.diff(lay["codes"][lay["order"]].astype(np.int64)) >= 0).all()


@pytest.mark.parametrize("bad", ["inf", "-inf", "nan_row", "signed_nan"])
def test_emulated_build_shows_the_non_finite_defect_and_its_fix(bad):
    """before the fix, one row with a non-finite coordinate gave every point the same Morton code on at least one axis (an
    infinite extent or an all-NaN row: every code 0), so the sort left the cloud in input order; with the fix the finite rows keep
    the codes and order of the finite cloud alone and the non-finite rows sort after them"""
    g = np.random.default_rng(5)
    fin = g.normal(0, 5, (4000, 3))
    row = {"inf": [np.inf, 0.0, 0.0], "-inf": [0.0, 0.0, -np.inf], "nan_row": [np.nan] * 3,
           "signed_nan": [0.0, np.copysign(np.nan, -1.0), 0.0]}[bad]
    pos = 1234
    p = np.insert(fin, pos, row, axis=0)
    old = R.tree_layout(p, fixed=False)
    if bad == "signed_nan":                                        # the NaN sorts below -inf: lo[y] is NaN, the y axis collapses
        assert np.isnan(old["lo"][1])
        y_bits = sum(1 << (3 * b + 1) for b in range(R.PC_BITS))
        assert (old["codes"] & np.uint32(y_bits) == 0).all()
    else:
        assert (old["codes"] == 0).all() and np.array_equal(old["order"], np.arange(p.shape[0]))
    new, ref = R.tree_layout(p), R.tree_layout(fin)
    assert np.array_equal(new["lo"], ref["lo"]) and np.array_equal(new["hi"], ref["hi"])
    keep = np.flatnonzero(np.arange(p.shape[0]) != pos)
    assert np.array_equal(new["codes"][keep], ref["codes"])
    assert np.array_equal(new["order"][:-1], keep[ref["order"]]) and new["order"][-1] == pos


def test_emulated_build_without_a_finite_row():
    p = np.array([[np.nan, 0.0, 0.0], [np.inf, -np.inf, 0.0], [np.nan] * 3])
    lay = R.tree_layout(p)
    assert np.isnan(lay["lo"]).all() and np.isnan(lay["hi"]).all()
    assert (lay["codes"] == 2 ** 30).all() and np.array_equal(lay["order"], [0, 1, 2])
