"""CPU checks of the edge inputs in rng_reference.py that test_gpu_device_rng_edges.py feeds the device streams: the exact log
oracle against the long-double estimate and glibc, the crafted attempt sets reaching the inputs they name, the word-level
Gaussian restatement against numpy, and the randperm patterns' closed-form round counts against the reservation model."""
import math

import numpy as np
import pytest
import torch

import rng_reference as R
from lidiff_b200 import _lib, rng


def test_cr_log_agrees_with_the_long_double_estimate_and_glibc():
    """cr_log's distance equals midpoint_distance to 2^-9 ulp, and glibc's log is cr_log's value wherever the distance exceeds
    the band"""
    _, _, r2, acc = R.attempts(R.words_for(*R.random_accepted(3000, 5)))
    near = R.attempts(R.words_for(*R.near_midpoint_attempts(n_cand=200_000, keep=2000, seed=7)))[2]
    crafted = [R.attempts(R.words_for(*s))[2] for s in (R.binade_attempts(), R.switch_attempts(), R.pow2_attempts())]
    x = np.concatenate([r2[acc], near] + crafted)
    y, d = R.cr_logs(x)
    md = R.midpoint_distance(x)
    ok = ~np.isnan(md)
    assert np.abs(d[ok] - md[ok]).max() < 2.0 ** -9
    assert (np.isnan(md) == R.is_pow2(np.log(x.astype(np.longdouble)).astype(np.float64))).all()
    libm = R.libm_log(x)
    outside = d > _lib.GAUSS_BAND
    assert outside.sum() > 3000 and np.array_equal(libm[outside], y[outside])
    assert (d <= 0.5).all()


@pytest.mark.parametrize("r2,log", [(0.5, -math.log(2)), (2.0 ** -104, -104 * math.log(2))])
def test_cr_log_of_known_values(r2, log):
    y, d = R.cr_log(r2)
    assert abs(y - log) <= math.ulp(log) and abs(d) <= 0.5


def test_cr_log_signs_the_distance():
    """the signed distance is positive when the exact log lies above the midpoint: the rounded value is then above it too"""
    x = R.attempts(R.words_for(*R.near_midpoint_attempts(n_cand=50_000, keep=200, seed=3)))[2]
    for v in x:
        y, d = R.cr_log(float(v))
        mid_below = d > 0
        nb = math.nextafter(y, -math.inf if mid_below else math.inf)
        assert abs(math.log(v) - y) <= abs(nb - y)           # glibc lands on y or its neighbour across that midpoint


def test_near_midpoint_set():
    """about 20 000 distinct accepted r2 within 2^-6 ulp of a midpoint, at least 100 of them within 2^-14, across the binades"""
    d1, d2 = R.near_midpoint_attempts()
    _, _, r2, acc = R.attempts(R.words_for(d1, d2))
    assert acc.all() and np.unique(r2).size == r2.size
    _, d = R.cr_logs(r2)
    assert 19_000 <= r2.size <= 20_000 and (d < 2.0 ** -6).all()
    assert (d < 2.0 ** -14).sum() >= 100
    assert np.unique(np.frexp(r2)[1]).size >= 90
    m = np.frexp(r2)[0]
    assert (m < 0.53).sum() >= 500                          # dd_log's largest |s| without the m < 1/sqrt(2) switch


def test_polar_edges_reach_what_they_name():
    r2 = {name: R.attempts(R.words_for(d1, d2))[2][0] for name, d1, d2, _ in R.polar_edges()}
    assert r2["r2_zero"] == 0.0 and r2["x1_minus_one"] == 1.0 and r2["r2_two"] == 2.0 and r2["r2_just_above_one"] > 1.0
    assert r2["smallest_r2"] == r2["smallest_r2_x2_negative"] == 2.0 ** -104
    assert r2["largest_r2"] == r2["largest_r2_negative"] == math.nextafter(1.0, 0.0)
    assert r2["x1_minus_one_plus_ulp"] == 1.0 - 2.0 ** -51
    for name, d1, d2, acc in R.polar_edges():
        x1, x2, _, a = R.attempts(R.words_for(d1, d2))
        assert bool(a[0]) == acc, name
        if name.endswith("negative"):
            assert x1[0] < 0 or x2[0] < 0
    signs = {(np.sign(x1[0]), np.sign(x2[0])) for x1, x2, _, _ in
             (R.attempts(R.words_for(d1, d2)) for name, d1, d2, _ in R.polar_edges() if name.startswith("quadrant"))}
    assert len(signs) == 4


def test_binade_switch_and_power_of_two_sets():
    _, _, r2, acc = R.attempts(R.words_for(*R.binade_attempts()))
    assert acc.all()
    j = 1 - np.frexp(r2)[1]
    assert np.array_equal(np.bincount(j)[1:], np.full(104, 3))
    assert np.array_equal(r2[0::3], 2.0 ** -np.arange(1, 105))          # every bottom exactly
    assert (r2[2::3][:40] == np.nextafter(2.0 ** -np.arange(0, 40), 0)).sum() >= 38

    _, _, r2, acc = R.attempts(R.words_for(*R.switch_attempts()))
    c0 = float.fromhex("0x1.6a09e667f3bcdp-1")                          # the double nearest 1/sqrt(2)
    assert acc.all() and r2.size == 85
    m = np.frexp(r2)[0]
    assert (m == c0).sum() == 5 and (m < c0).sum() == 40 and np.abs((m - c0) / np.spacing(c0)).max() == 8

    _, _, r2, acc = R.attempts(R.words_for(*R.pow2_attempts()))
    y, _ = R.cr_logs(r2)
    assert acc.all()
    for p in R.POW2_LOGS:
        assert (y > p).any() and (y < p).any()
        assert np.isin([math.nextafter(p, 0.0), math.nextafter(p, -1.0)], y).all() or (y == p).any()
    assert (y == -1.0).any() and (y == -2.0).any()


def test_rejection_stream_accepts_one_attempt_in_a_thousand():
    d1, d2 = R.rejection_stream()
    _, _, r2, acc = R.attempts(R.words_for(d1, d2))
    assert np.array_equal(np.flatnonzero(acc), np.arange(999, 256_000, 1000))
    assert {0.0, 1.0, 2.0} <= set(r2[~acc].tolist())
    out, info = R.gauss_from_words(R.words_for(d1, d2), 512)
    assert info["words_used"] == 4 * 256_000 and not info["short_words"]
    assert R.gauss_from_words(R.words_for(d1, d2)[:-4], 512)[1]["short_words"] == 1


@pytest.mark.parametrize("n_out,cached", [(0, True), (1, True), (2, True), (1, False), (2, False), (7, False), (30, True)])
def test_gauss_from_words_equals_numpy(n_out, cached):
    """the word-level restatement against numpy from a state that emits the same words (polar edges, then random attempts)"""
    e = R.polar_edges()
    a1, a2 = R.random_accepted(40, 11)
    words = R.words_for(np.concatenate([[x[1] for x in e], a1]), np.concatenate([[x[2] for x in e], a2]))
    rs = R.crafted_state(words, cached, 0.375)
    assert np.array_equal(R.mt_words(rs.get_state(legacy=True)[1], R.MT_N - words.size, words.size)[0], words)
    ref = rs.randn(n_out)
    _, _, pos, hg, g = rs.get_state(legacy=True)
    out, info = R.gauss_from_words(words, n_out, int(cached), 0.375)
    assert np.array_equal(out.view(np.uint64), ref.view(np.uint64))
    assert info["has_gauss"] == hg and info["gauss"] == g and R.MT_N - words.size + info["words_used"] == pos


@pytest.mark.parametrize("pattern", list(R.RANDPERM_PATTERNS))
def test_randperm_patterns_closed_forms(pattern):
    make, closed = R.RANDPERM_PATTERNS[pattern]
    for n in list(range(2, 41)) + [257, 1000]:
        words = make(n)
        perm, rounds = R.randperm_rounds(words, n)
        assert np.array_equal(perm, R.fisher_yates(words, n)), n
        if closed is not None:
            assert rounds == closed(n), n


@pytest.mark.parametrize("n", [0, 1, 2, 3, 624, 5000])
def test_fisher_yates_equals_torch(n):
    g = torch.Generator().manual_seed(n)
    key, pos = rng.torch_state_decode(g.get_state())
    words, _, _ = R.mt_words(key, pos, max(n - 1, 0))
    assert np.array_equal(R.fisher_yates(words, n), torch.randperm(n, generator=g).numpy())
