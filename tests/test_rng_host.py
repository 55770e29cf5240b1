"""CPU checks of the device random streams' contracts (csrc/rng.cu, lidiff_b200/rng.py): the numpy restatements in
rng_reference.py against np.random.randn and torch.randperm, torch's state layout, glibc's log against the band, crafted numpy
states that reach the polar method's edges."""
import math

import numpy as np
import pytest
import torch

import rng_reference as R
from lidiff_b200 import _lib, rng


def _np_state(seed, burn=0):
    rs = np.random.RandomState(seed)
    if burn:
        rs.randn(burn)
    return rs


@pytest.mark.parametrize("seed,burn,n", [(0, 0, 1), (1, 0, 2), (2, 3, 3), (3, 0, 1247), (4, 1, 1248), (5, 7, 20001), (6, 311, 5)])
def test_legacy_gauss_restatement_equals_numpy(seed, burn, n):
    rs = _np_state(seed, burn)
    _, key, pos, hg, g = rs.get_state(legacy=True)
    out, key2, pos2, hg2, g2, used, _ = R.legacy_gauss(key, pos, hg, g, n)
    ref = rs.randn(n)
    assert np.array_equal(out.view(np.uint64), ref.view(np.uint64))
    _, k, p, h, c = rs.get_state(legacy=True)
    assert np.array_equal(k, key2) and p == pos2 and h == hg2 and c == g2


def test_mt_phases_equal_numpy_words():
    """the three-phase twist gives numpy's words over several twists, from every kind of position"""
    for seed, pos_draws in [(0, 0), (9, 1), (10, 623), (11, 624)]:
        rs = np.random.RandomState(seed)
        rs.randint(0, 2 ** 32, size=pos_draws, dtype=np.uint32)
        _, key, pos, _, _ = rs.get_state(legacy=True)
        words, key2, pos2 = R.mt_words(key, pos, 2000)
        assert np.array_equal(words, rs.randint(0, 2 ** 32, size=2000, dtype=np.uint32))
        _, k, p, _, _ = rs.get_state(legacy=True)
        assert np.array_equal(k, key2) and p == pos2


def test_untemper_inverts_temper():
    w = np.random.RandomState(3).randint(0, 2 ** 32, size=100000, dtype=np.uint32)
    assert np.array_equal(rng.untemper(R.temper(w)), w)


def test_state_after_from_emitted_words():
    """rng._state_after recovers numpy's key and pos after any number of used words, from the emitted words alone"""
    rs = np.random.RandomState(12)
    rs.randn(101)
    _, key, pos, _, _ = rs.get_state(legacy=True)
    nw = 4000
    words, key_end, _ = R.mt_words(key, pos, nw)
    for used in [0, 1, 4, 624 - pos, 624 - pos + 1, 1247, 1248 + 624 - pos, nw - 1, nw]:
        k, p = rng._state_after(key, pos, used, torch.from_numpy(words.view(np.int32)), nw, torch.from_numpy(key_end.view(np.int32)))
        _, k_ref, p_ref = R.mt_words(key, pos, used)
        assert np.array_equal(k, k_ref) and p == p_ref, used


@pytest.mark.parametrize("n", [0, 1, 2, 623, 624, 625, 5000])
@pytest.mark.parametrize("draws", [0, 1, 622, 700])
def test_randperm_rounds_equal_torch(n, draws):
    g = torch.Generator().manual_seed(n + draws)
    if draws:
        torch.randperm(draws + 1, generator=g)                # draws words: a mid-block state
    key, pos = rng.torch_state_decode(g.get_state())
    words, key2, pos2 = R.mt_words(key, pos, max(n - 1, 0))
    perm, _ = R.randperm_rounds(words, n)
    assert np.array_equal(perm, R.fisher_yates(words, n))
    assert np.array_equal(perm, torch.randperm(n, generator=g).numpy())
    if n >= 2:
        k, p = rng.torch_state_decode(g.get_state())
        assert np.array_equal(k, key2) and p == pos2


def test_randperm_rounds_at_200003():
    g = torch.Generator().manual_seed(7)
    key, pos = rng.torch_state_decode(g.get_state())
    words, _, _ = R.mt_words(key, pos, 200002)
    perm, rounds = R.randperm_rounds(words, 200003)
    assert np.array_equal(perm, torch.randperm(200003, generator=g).numpy())
    assert rounds < 64


def test_torch_state_round_trip():
    torch.manual_seed(3)
    torch.randperm(1000)
    s = torch.get_rng_state()
    key, pos = rng.torch_state_decode(s)
    s2 = rng.torch_state_encode(s, key, pos)
    assert torch.equal(s, s2)
    torch.set_rng_state(s2)
    a = torch.randperm(5000)
    torch.set_rng_state(s)
    assert torch.equal(a, torch.randperm(5000))
    torch.manual_seed(4)                                       # fresh: left 1, next 0
    key, pos = rng.torch_state_decode(torch.get_rng_state())
    assert pos == 624


def test_torch_state_refuses_unknown_layouts():
    s = torch.get_rng_state()
    with pytest.raises(ValueError):
        rng.torch_state_decode(s[:-8])
    bad = s.clone()
    bad[8:12] = torch.tensor([0, 4, 0, 0], dtype=torch.uint8)          # left = 1024
    with pytest.raises(ValueError):
        rng.torch_state_decode(bad)


def test_refusals_before_any_device_work():
    with pytest.raises(TypeError, match="Generator"):
        rng.numpy_randn(3, random_state=np.random.default_rng(0))
    with pytest.raises(ValueError, match="2\\^32 / 20"):
        rng.torch_randperm(_lib.RANDPERM_MAX_N)


def test_libm_log_is_correctly_rounded_outside_the_band():
    """glibc's log (which numpy's legacy_gauss and math.log call) returns the correctly rounded value wherever the exact log lies
    more than LB2_GAUSS_BAND ulp from a rounding midpoint: 10^6 accepted r2 of the polar method and inputs next to midpoints"""
    rs = np.random.RandomState(2024)
    _, key, pos, _, _ = rs.get_state(legacy=True)
    words, _, _ = R.mt_words(key, pos, 4 * 1_300_000)
    _, _, r2, acc = R.attempts(words)
    r2 = r2[acc][:1_000_000]
    assert r2.size == 1_000_000
    # inputs whose log lies near a midpoint: scan neighbours of many r2 and keep those closest
    base = np.random.RandomState(5).uniform(1e-6, 1.0, 20000)
    near = (base[:, None] + np.arange(-64, 64)[None, :] * np.spacing(base)[:, None]).ravel()
    dn = R.midpoint_distance(near)
    near = near[np.argsort(np.nan_to_num(dn, nan=1.0))[:20000]]
    x = np.concatenate([r2, near, [np.nextafter(1.0, 0.0), 2.0 ** -104, 0.5, 0.25]])
    libm = np.array([math.log(v) for v in x])
    cr = np.log(x.astype(np.longdouble)).astype(np.float64)
    d = R.midpoint_distance(x)
    outside = d > _lib.GAUSS_BAND
    assert (libm[outside] == cr[outside]).all()
    frac = float((~outside[: r2.size]).mean())
    assert 0.03 < frac < 0.10, frac                                  # about 2 x band of the accepted attempts
    assert (dn < 0.01).sum() > 100                                   # the constructed inputs do reach the band


@pytest.mark.parametrize("case,d1,d2,accepted", [
    ("r2_zero", 1 << 52, 1 << 52, False),                      # x1 = x2 = 0
    ("x_minus_one", 0, 1 << 52, False),                        # x1 = -1, x2 = 0: r2 = 1
    ("r2_ge_one", 0, 0, False),                                # r2 = 2
    ("smallest_r2", (1 << 52) + 1, 1 << 52, True),             # x1 = 2^-52: r2 = 2^-104
    ("largest_r2", 1, 1 << 52, True),                          # x1 = -1 + 2^-52: r2 just below 1
])
def test_crafted_states_reach_the_polar_edges(case, d1, d2, accepted):
    rs = R.crafted_state(R.words_for(d1, d2))
    _, key, pos, hg, g = rs.get_state(legacy=True)
    words, _, _ = R.mt_words(key, pos, 4)
    x1, x2, r2, acc = R.attempts(words)
    assert bool(acc[0]) == accepted, (x1, x2, r2)
    out, key2, pos2, hg2, g2, used, _ = R.legacy_gauss(key, pos, hg, g, 3)
    ref = rs.randn(3)
    assert np.array_equal(out.view(np.uint64), ref.view(np.uint64))
    assert (R.legacy_gauss(key, pos, hg, g, 1)[5] == 4) == accepted     # one output: the first attempt serves it iff accepted
    _, k, p, h, c = rs.get_state(legacy=True)
    assert np.array_equal(k, key2) and p == pos2 and h == hg2 and c == g2
