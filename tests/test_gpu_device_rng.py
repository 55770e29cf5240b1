"""numpy_randn / torch_randperm on the H100 against np.random.randn / torch.randperm, bit for bit, and the host generators' states
afterwards (lidiff_b200/rng.py, csrc/rng.cu)."""
import numpy as np
import pytest
import torch

from lidiff_b200 import _lib, rng

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _state_eq(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:4] == b[2:4] and a[4] == b[4]


def _check_randn(rs_dev, rs_host, shape, band=_lib.GAUSS_BAND):
    got = rng.numpy_randn(*shape, device=DEV, random_state=rs_dev, band=band)
    ref = rs_host.randn(*shape)
    assert tuple(got.shape) == np.shape(ref)
    assert np.array_equal(got.cpu().numpy().view(np.uint64), np.asarray(ref).view(np.uint64))
    assert _state_eq(rs_dev.get_state(legacy=True), rs_host.get_state(legacy=True))


def _pair(seed, pre=0, pre_odd=False, pos_words=0):
    """two RandomStates in the same state: `pre` values drawn (odd: a cached Gaussian), or `pos_words` raw words drawn"""
    out = []
    for _ in range(2):
        rs = np.random.RandomState(seed)
        if pos_words:
            rs.randint(0, 2 ** 32, size=pos_words, dtype=np.uint32)
        if pre:
            rs.randn(pre + (1 if pre_odd else 0))
        out.append(rs)
    return out


SIZES = [0, 1, 2, 3, 311, 312, 313, 623, 624, 625, 1247, 1248, 1249]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("cached", [False, True])
def test_randn_sizes_with_and_without_a_cached_gaussian(n, cached):
    a, b = _pair(11 + n, pre=4, pre_odd=cached)
    assert a.get_state(legacy=True)[3] == int(cached)
    _check_randn(a, b, (n,))


@pytest.mark.parametrize("pos_words", [0, 1, 300, 623, 624])
@pytest.mark.parametrize("seed", [0, 1, 12345])
def test_randn_from_every_position(pos_words, seed):
    a, b = _pair(seed, pos_words=pos_words)
    _check_randn(a, b, (2, 500, 3))


def test_randn_at_the_refinement_sample_size_and_the_global_generator():
    np.random.seed(7)
    np.random.randn(5)                                            # interleaved host draws before ...
    b = np.random.RandomState()
    b.set_state(np.random.get_state())
    got = rng.numpy_randn(1, 4146667, 3, device=DEV)              # 12 440 001 values
    ref = b.randn(1, 4146667, 3)
    assert np.array_equal(got.cpu().numpy().view(np.uint64), ref.view(np.uint64))
    assert _state_eq(np.random.get_state(legacy=True), b.get_state(legacy=True))
    assert np.array_equal(np.random.randn(7), b.randn(7))         # ... and after


@pytest.mark.parametrize("n", [1, 2, 3, 1001, 100001])
def test_randn_all_deferred_band_gives_the_same_bits(n):
    a, b = _pair(3, pre=1, pre_odd=bool(n & 1))
    _check_randn(a, b, (n,), band=0.5)
    st = {}
    c, d = _pair(4)
    rng.numpy_randn(n, device=DEV, random_state=c, band=0.5, stats=st)
    assert st["deferred"] == st["pairs"]


def test_randn_reruns_give_the_same_bits_and_defer_about_two_bands():
    outs = []
    for _ in range(2):
        a, _ = _pair(99)
        st = {}
        outs.append(rng.numpy_randn(1000000, device=DEV, random_state=a, stats=st).cpu())
        frac = st["deferred"] / st["pairs"]
        assert 0.03 < frac < 0.10, frac
    assert torch.equal(outs[0], outs[1])


def test_randn_refuses_a_generator():
    with pytest.raises(TypeError, match="Generator"):
        rng.numpy_randn(3, device=DEV, random_state=np.random.default_rng(0))


def _gen_pair(seed, draws):
    gens = [torch.Generator().manual_seed(seed) for _ in range(2)]
    for g in gens:
        if draws:
            torch.randperm(draws + 1, generator=g)
    return gens


@pytest.mark.parametrize("n", [0, 1, 2, 623, 624, 625, 100000, 4146667])
@pytest.mark.parametrize("draws", [0, 300])
def test_randperm_equals_torch(n, draws):
    a, b = _gen_pair(n + 1, draws)
    got = rng.torch_randperm(n, device=DEV, generator=a)
    ref = torch.randperm(n, generator=b)
    assert got.dtype == torch.int64 and torch.equal(got.cpu(), ref)
    assert torch.equal(a.get_state(), b.get_state())


def test_randperm_default_generator_reruns_and_rounds():
    torch.manual_seed(5)
    s = torch.get_rng_state()
    st = {}
    got = rng.torch_randperm(1036666, device=DEV, stats=st)
    after = torch.get_rng_state()
    torch.set_rng_state(s)
    assert torch.equal(got.cpu(), torch.randperm(1036666))
    assert torch.equal(after, torch.get_rng_state())
    torch.set_rng_state(s)
    assert torch.equal(rng.torch_randperm(1036666, device=DEV).cpu(), got.cpu())
    assert 1 <= st["rounds"] < 64


def test_randperm_refuses_64_bit_draws():
    with pytest.raises(ValueError, match="2\\^32 / 20"):
        rng.torch_randperm(_lib.RANDPERM_MAX_N, device=DEV)
    h = _lib.get_handle(DEV)
    with pytest.raises(RuntimeError, match="2\\^32 / 20"):
        h.randperm(None, _lib.RANDPERM_MAX_N, None)

