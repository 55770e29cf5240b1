"""The device random streams (csrc/rng.cu) at their edges on the H100, with words injected straight into the kernels:

- lb2_legacy_gauss over crafted attempts (rng_reference: polar edges, every binade of r2, the m < 1/sqrt(2) switch, logs at and
  next to powers of two, logs within 2^-6 ulp of a rounding midpoint, rejection-heavy streams) against numpy's formula with
  glibc's log, and, at narrower bands, against the correctly rounded log (cr_log): dd_log's error bound checked directly;
- lb2_randperm on reservation patterns that need n - 1 rounds or give every thread several iterations, against sequential
  Fisher-Yates and the reservation model's round count;
- lb2_mt19937_words from every phase boundary of the twist, and over 10^8 words, against numpy's MT19937.
"""
import numpy as np
import pytest
import torch

import rng_reference as R
from lidiff_b200 import _lib, rng

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BAND = _lib.GAUSS_BAND
TOL = 2.0 ** -14        # dd_log's claim (relative error below 2^-68) is at most 2^-15 ulp: the margin taken either side of a band
SETS = ["polar_edges", "binades", "switch", "pow2", "near_midpoint", "rejection_heavy"]
EDGES = R.polar_edges()


@pytest.fixture(scope="module")
def h():
    return _lib.get_handle(DEV)


@pytest.fixture(scope="module")
def attempt_sets():
    return {
        "polar_edges": (np.array([e[1] for e in EDGES]), np.array([e[2] for e in EDGES])),
        "binades": R.binade_attempts(),
        "switch": R.switch_attempts(),
        "pow2": R.pow2_attempts(),
        "near_midpoint": R.near_midpoint_attempts(),
        "rejection_heavy": R.rejection_stream(),
    }


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _dev_words(words):
    words = np.asarray(words, np.uint32)
    return torch.from_numpy(np.ascontiguousarray(words if words.size else np.zeros(4, np.uint32)).view(np.int32)).to(DEV)


def _gauss(h, words, n_out, has_gauss=0, gauss=0.0, band=BAND, n_words=None):
    out = torch.empty(max(n_out, 1), dtype=torch.float64, device=DEV)
    info = h.legacy_gauss(_dev_words(words), len(words) if n_words is None else n_words, n_out, has_gauss, gauss, band, out)
    return out[:n_out].cpu().numpy(), info


def _cr(r2):
    return R.cr_logs(r2)[0]


def _classes(r2, band):
    """(leading word certain, libm certain) per accepted attempt: the exact log lies more than band + TOL ulp from the midpoint (and
    the result is not a power of two), or within band - TOL ulp of it (or the result is a power of two)"""
    y, d = R.cr_logs(r2)
    p2 = R.is_pow2(y)
    return (d > band + TOL) & ~p2, (d < band - TOL) | p2


# ---- legacy Gaussian ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SETS)
def test_gauss_at_the_default_band_equals_numpy_formula(h, attempt_sets, name):
    """band = LB2_GAUSS_BAND: every output is numpy's f x2 / f x1 with glibc's log, bit for bit; the Lb2GaussInfo fields are exact,
    and the deferred count lies between the counts at band -+ 2^-14 ulp"""
    words = R.words_for(*attempt_sets[name])
    n_out = 2 * int(R.attempts(words)[3].sum())
    got, info = _gauss(h, words, n_out)
    ref, ri = R.gauss_from_words(words, n_out)
    assert np.array_equal(_bits(got), _bits(ref)), f"{int((_bits(got) != _bits(ref)).sum())} of {n_out} outputs differ"
    assert (info.words_used, info.short_words, info.has_gauss, info.gauss) == (ri["words_used"], 0, 0, 0.0)
    leading, libm = _classes(ri["r2"], BAND)
    assert libm.sum() <= info.deferred <= (~leading).sum()


@pytest.mark.parametrize("band", [0.0, 2.0 ** -12, 2.0 ** -6])
@pytest.mark.parametrize("name", SETS)
def test_gauss_outside_the_band_gives_the_correctly_rounded_log(h, attempt_sets, name, band):
    """at narrower bands the leading word of dd_log decides attempts close to a midpoint: every attempt more than band + 2^-14 ulp
    from it gives the output of the correctly rounded log, and every deferred one the output of glibc's"""
    words = R.words_for(*attempt_sets[name])
    n_out = 2 * int(R.attempts(words)[3].sum())
    got, info = _gauss(h, words, n_out, band=band)
    cr, ri = R.gauss_from_words(words, n_out, log=_cr)
    libm, _ = R.gauss_from_words(words, n_out)
    leading, host = (np.repeat(c, 2) for c in _classes(ri["r2"], band))
    g, c, m = _bits(got), _bits(cr), _bits(libm)
    wrong = leading & (g != c)
    assert not wrong.any(), (f"{int(wrong.sum())} outputs differ from the correctly rounded log's, first at r2 = "
                             f"{ri['r2'][np.flatnonzero(wrong)[0] // 2]!r}")
    assert not (host & (g != m)).any()
    assert ((g == c) | (g == m)).all()
    assert host[::2].sum() <= info.deferred <= (~leading[::2]).sum()
    assert info.words_used == ri["words_used"] and not info.short_words


@pytest.fixture(scope="module")
def far_and_near(attempt_sets):
    """(d1, d2) of 20 accepted attempts more than band + 2^-14 ulp from a midpoint, and of one within band - 2^-14 ulp"""
    d1, d2 = attempt_sets["binades"]
    leading, _ = _classes(R.attempts(R.words_for(d1, d2))[2], BAND)
    far = np.flatnonzero(leading)[:20]
    n1, n2 = attempt_sets["near_midpoint"]
    return (d1[far], d2[far]), (n1[:1], n2[:1])


@pytest.mark.parametrize("cached", [False, True])
@pytest.mark.parametrize("last_deferred", [False, True])
def test_trailing_gaussian_equals_numpy(h, far_and_near, last_deferred, cached):
    """an odd count: the trailing f x1 of the last attempt becomes numpy's cached Gaussian, whether that attempt's log was resolved
    on the device or on the host"""
    (f1, f2), (n1, n2) = far_and_near
    last = (n1, n2) if last_deferred else (f1[-1:], f2[-1:])
    words = R.words_for(np.concatenate([f1[:-1], last[0]]), np.concatenate([f2[:-1], last[1]]))
    n_out = 2 * 20 - 1 + int(cached)
    rs = R.crafted_state(words, cached, 0.625)
    ref = rs.randn(n_out)
    _, key, pos, hg, g = rs.get_state(legacy=True)
    got, info = _gauss(h, words, n_out, int(cached), 0.625)
    assert np.array_equal(_bits(got), _bits(ref))
    assert info.has_gauss == hg == 1 and _bits(info.gauss) == _bits(g)
    assert info.deferred == int(last_deferred)
    assert info.words_used == len(words) and pos == R.MT_N


@pytest.mark.parametrize("n_out,cached", [(1, True), (2, True), (3, True), (1, False), (2, False)])
def test_small_counts_and_the_cached_gaussian(h, n_out, cached):
    """n_out = 1 with a cached value returns it and clears the cache; 2 uses it and caches the next pair's f x1"""
    words = R.words_for([e[1] for e in EDGES], [e[2] for e in EDGES])
    rs = R.crafted_state(words, cached, -1.75)
    start = R.MT_N - len(words)
    ref = rs.randn(n_out)
    _, _, pos, hg, g = rs.get_state(legacy=True)
    got, info = _gauss(h, words, n_out, int(cached), -1.75)
    assert np.array_equal(_bits(got), _bits(ref))
    assert info.has_gauss == hg and _bits(info.gauss) == _bits(g)
    assert start + info.words_used == pos


def test_rejection_heavy_streams(h, attempt_sets):
    """one accepted attempt in 1000: the last needed attempt is the array's last, so words_used is every word; one attempt (or one
    word) fewer, or fewer attempts than pairs, gives short_words = 1"""
    words = R.words_for(*attempt_sets["rejection_heavy"])
    pairs = 256
    for n_out in (2 * pairs, 2 * pairs - 1):
        got, info = _gauss(h, words, n_out)
        ref, ri = R.gauss_from_words(words, n_out)
        assert np.array_equal(_bits(got), _bits(ref))
        assert info.words_used == len(words) == ri["words_used"] and not info.short_words
        assert info.has_gauss == n_out % 2 and _bits(info.gauss) == _bits(ri["gauss"])
    for n_words in (len(words) - 4, len(words) - 1, 4 * (pairs - 1)):
        _, info = _gauss(h, words, 2 * pairs, n_words=n_words)
        assert info.short_words == 1 == R.gauss_from_words(words[:n_words], 2 * pairs)[1]["short_words"]
        assert info.words_used == 0


@pytest.mark.parametrize("n", [1, 3, 6])
@pytest.mark.parametrize("edge", EDGES, ids=[e[0] for e in EDGES])
def test_numpy_randn_from_crafted_states(edge, n):
    """rng.numpy_randn from a state whose next attempt is a polar edge: numpy's values and numpy's state afterwards"""
    _, d1, d2, _ = edge
    a, b = (R.crafted_state(R.words_for(d1, d2)) for _ in range(2))
    got = rng.numpy_randn(n, device=DEV, random_state=a)
    ref = b.randn(n)
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(ref))
    sa, sb = a.get_state(legacy=True), b.get_state(legacy=True)
    assert np.array_equal(sa[1], sb[1]) and sa[2:4] == sb[2:4] and _bits(sa[4]) == _bits(sb[4])


# ---- randperm ------------------------------------------------------------------------------------------------------------------
def _grid_threads():
    """the threads the cooperative randperm grid can hold: every SM's resident-thread limit (k_randperm's 32 registers fit 8 CTAs
    of 256 per SM, which is that limit on the H100)"""
    p = torch.cuda.get_device_properties(DEV)
    return p.multi_processor_count * p.max_threads_per_multi_processor


def _randperm(h, words, n):
    out = torch.empty(n, dtype=torch.int64, device=DEV)
    rounds = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    h.randperm(_dev_words(words), n, out, rounds)
    return out.cpu().numpy(), int(rounds.item())


@pytest.mark.parametrize("n", [2, 3, 257, 65537])
@pytest.mark.parametrize("pattern", ["last_slot", "chain"])
def test_randperm_patterns_of_n_minus_one_rounds(h, pattern, n):
    """every iteration aims at the last slot, or waits for its predecessor: one iteration closes per round"""
    words = R.RANDPERM_PATTERNS[pattern][0](n)
    got, rounds = _randperm(h, words, n)
    assert np.array_equal(got, R.fisher_yates(words, n))
    assert rounds == n - 1
    if n <= 257:
        assert rounds == R.randperm_rounds(words, n)[1]


@pytest.mark.parametrize("size", ["small", "grid_plus_1", "grid_plus_2", "4M"])
@pytest.mark.parametrize("pattern", ["zeros", "odd_one", "even_one", "all_ones", "small_z"])
def test_randperm_patterns_of_few_rounds(h, pattern, size):
    """patterns that close in a few rounds, at sizes where threads own several iterations: just above the grid's thread count, and
    4 M; the rounds are the closed form where there is one, else the reservation model's"""
    g = _grid_threads()
    sizes = {"small": [2, 3, 4, 5, 257], "grid_plus_1": [g + 1], "grid_plus_2": [g + 2], "4M": [4_000_037]}[size]
    make, closed = R.RANDPERM_PATTERNS[pattern]
    for n in sizes:
        words = make(n)
        got, rounds = _randperm(h, words, n)
        assert np.array_equal(got, R.fisher_yates(words, n)), n
        if closed is not None:
            assert rounds == closed(n), n
        if closed is None or n <= 257:
            assert rounds == R.randperm_rounds(words, n)[1], n


# ---- MT19937 words -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 227, 228, 454, 455, 623, 624, 625, 1248])
@pytest.mark.parametrize("pos", [0, 1, 226, 227, 453, 454, 623, 624])
def test_mt19937_words_across_the_twist_phases(h, pos, n):
    """the words, the state written back and pos_out from every phase boundary of the twist, against mt_words and RandomState;
    nothing past n is written"""
    key = np.random.RandomState(1000 * pos + n).get_state(legacy=True)[1]
    state = torch.from_numpy(key.view(np.int32).copy()).to(DEV)
    out = torch.full((n + 64,), 0x5A5A5A5A, dtype=torch.int32, device=DEV)
    pos_out = h.mt19937_words(state, pos, n, out)
    words, key2, pos2 = R.mt_words(key, pos, n)
    got = out.cpu().numpy().view(np.uint32)
    assert np.array_equal(got[:n], words) and (got[n:] == 0x5A5A5A5A).all()
    assert np.array_equal(state.cpu().numpy().view(np.uint32), key2) and pos_out == pos2
    rs = np.random.RandomState()
    rs.set_state(("MT19937", key, pos, 0, 0.0))
    assert np.array_equal(rs.randint(0, 2 ** 32, size=n, dtype=np.uint32), words)
    _, k, p, _, _ = rs.get_state(legacy=True)
    assert np.array_equal(k, key2) and p == pos2


def test_mt19937_words_over_10_to_the_8(h):
    rs = np.random.RandomState(77)
    rs.randint(0, 2 ** 32, size=300, dtype=np.uint32)
    _, key, pos, _, _ = rs.get_state(legacy=True)
    state = torch.from_numpy(key.view(np.int32).copy()).to(DEV)
    n = 10 ** 8
    out = torch.empty(n, dtype=torch.int32, device=DEV)
    pos_out = h.mt19937_words(state, pos, n, out)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), rs.randint(0, 2 ** 32, size=n, dtype=np.uint32))
    _, k, p, _, _ = rs.get_state(legacy=True)
    assert np.array_equal(state.cpu().numpy().view(np.uint32), k) and pos_out == p


# ---- the largest randperm ------------------------------------------------------------------------------------------------------
def test_randperm_at_the_largest_n_equals_torch():
    """The slowest test of this file.  rng.torch_randperm(RANDPERM_MAX_N - 1) against torch.randperm, and the generator states
    afterwards.  It holds two 1.7 GB permutations and torch's own working copy on the host: about 5 GB of host memory."""
    n = _lib.RANDPERM_MAX_N - 1
    a, b = (torch.Generator().manual_seed(20) for _ in range(2))
    got = rng.torch_randperm(n, device=DEV, generator=a).cpu()
    ref = torch.randperm(n, generator=b)
    assert torch.equal(got, ref)
    del got, ref
    assert torch.equal(a.get_state(), b.get_state())
