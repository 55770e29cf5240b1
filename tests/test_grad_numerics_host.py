"""The weight gradient's bars (tests/grad_numerics.py) have teeth, checked without a GPU: an emulation of lb2_spconv_wgrad's FP16x3
products (restated split of X and of G 2^k, fp32 sums per chunk, chunk partials added in order) passes both bars on every case;
holding G in one fp16, or dropping x_lo g_hi, fails the statistical bar; splitting G without its pre-scale fails the hard bar.  At
the row count of the golden scan the hard-only bar the weight-gradient test used before passes the FP16x2 mutant."""
import math
import os

import numpy as np
import pytest
import torch

import grad_numerics as gn
import split_numerics as sn

HERE = os.path.dirname(os.path.abspath(__file__))

# m_out, m_in, cin, cout, kvol, p (X ~ 2^p randn), max|G|, neighbour density
CASES = [(1, 1, 8, 32, 1, 0, 1e-4, 1.0), (65, 300, 16, 32, 8, 0, 1e-4, 0.7), (321, 500, 40, 64, 8, 0, 1e-4, 0.5),
         (8193, 9000, 32, 32, 8, 0, 1e-4, 0.4), (20000, 20000, 64, 64, 1, 0, 1e-4, 1.0), (4096, 4096, 96, 96, 8, -12, 1.0, 0.6),
         (4096, 4096, 16, 64, 8, 8, 1e-6, 0.6), (16384, 16384, 3, 32, 8, 0, 1e-4, 0.3), (6000, 6000, 5, 96, 8, -4, 1e6, 0.5)]
MUTANT_CASES = [c for c in CASES if c[0] >= 321 and c[5] >= -4]      # below 2^-4 the 2^-25 floor hides a dropped term by design


def case_id(c):
    m, m_in, cin, cout, kvol, p, gmax, dens = c
    return f"m{m}_{cin}to{cout}_k{kvol}_p{p}_g{gmax:g}"


_CACHE = {}


def _case(c):
    if c not in _CACHE:
        m, m_in, cin, cout, kvol, p, gmax, dens = c
        seed = m * 7 + cin * 131 + cout + kvol
        X, G = gn.operands(m_in, m, cin, cout, p, gmax, seed)
        nbr = None if kvol == 1 and m_in == m else gn.random_nbr(m, m_in, kvol, dens, seed + 1)
        _CACHE[c] = (X, G, nbr, gn.WgradReference(X, G, nbr, kvol))
    return _CACHE[c]


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_fp16x3_emulation_passes_both_bars(c):
    X, G, nbr, ref = _case(c)
    eh, es = ref.errors(gn.emulate_wgrad(X, G, nbr, c[4]))
    t = gn.tau_s(c[0])
    print(f"{case_id(c)}: hard {eh:.3f} of bound, stat {es:.2e} (tau_s {t:.2e})")
    assert eh <= 1.0
    assert es <= t


@pytest.mark.parametrize("scheme", ["f16x2", "no_xlo_ghi"])
@pytest.mark.parametrize("c", MUTANT_CASES, ids=case_id)
def test_cheaper_splits_fail_the_statistical_bar(c, scheme):
    X, G, nbr, ref = _case(c)
    _, es = ref.errors(gn.emulate_wgrad(X, G, nbr, c[4], scheme))
    t = gn.tau_s(c[0])
    print(f"{case_id(c)} {scheme}: stat {es:.2e} = {es / t:.1f} x tau_s")
    assert es > t


@pytest.mark.parametrize("gmax", [1e-4, 1e-6])
def test_unscaled_g_fails_the_hard_bar(gmax):
    c = (4096, 4096, 32, 64, 8, 0, gmax, 0.5)
    X, G, nbr, ref = _case(c)
    eh, _ = ref.errors(gn.emulate_wgrad(X, G, nbr, 8, "unscaled"))
    print(f"max|G| {gmax:g} unscaled: hard {eh:.1f} x bound")
    assert eh > 1.0


def test_hard_only_bar_misses_fp16x2_at_the_golden_scans_row_count():
    """the bar of the earlier weight-gradient test (tau S1 + floor, tau with ceil(m / 320) + 16 adds) on the golden scan's level-1
    map (18 000 rows, every one its own voxel): the FP16x2 emulation passes it, the statistical bar rejects it"""
    from oracle import me_cpu as ome
    z = np.load(os.path.join(HERE, "golden", "step_000123.npz"))
    pts = torch.from_numpy(z["part"]).float()
    geom = ome.TensorField(pts, torch.cat([torch.zeros(pts.shape[0], 1), torch.round(pts / 0.05)], 1)).sparse().geom
    m = geom.stride_level(1).shape[0]
    X, G = gn.operands(m, m, 32, 64, 0, 1e-4, 5)
    ref = gn.WgradReference(X, G, None, 1)
    dw = gn.emulate_wgrad(X, G, None, 1, "f16x2").double()
    err = (dw - ref.y).abs()
    tau_old = 3.002 * 2.0 ** -22 + 60 * 2.0 ** -23 + (math.ceil(m / 320) + 16) * 2.0 ** -24
    old = (err / (tau_old * ref.S1 + ref.floor)).max().item()
    _, es = ref.errors(dw)
    print(f"golden scan, {m} rows, 32 -> 64, FP16x2: earlier hard bar {old:.2f} of bound, statistical {es / gn.tau_s(m):.1f} x tau_s")
    assert old <= 1.0
    assert es > gn.tau_s(m)


def test_chunking_follows_the_kernel():
    assert [gn.nchunks_of(m) for m in (0, 1, 8192, 8193, 131072, 131073, 10 ** 6)] == [1, 1, 1, 2, 16, 16, 16]
    assert [gn.rows_per_chunk_of(m) for m in (1, 64, 65, 8193, 131073)] == [64, 64, 128, 4160, 8256]
    assert gn.chain(1) == (12, 1) and gn.chain(320) == (60, 1) and gn.chain(321) == (60, 2)
    assert gn.chain(131073) == (60, 26 + 15)


def test_edge_activations_below_the_split_limit_hold_the_representation_bound():
    """the X values of the GPU magnitude sweep: every finite edge value below 131024 splits within 2^-22 |x| + 2^-25"""
    e = sn.edge_values()
    e = e[torch.isfinite(e) & (e.abs() < gn.SPLIT_INF)]
    hi, lo = sn.split(e)
    err = (hi.double() + lo.double() - e.double()).abs()
    assert (err <= 2.0 ** -22 * e.double().abs() + 2.0 ** -25).all()


def test_sequential_restatement_is_ordered():
    """the row-sum restatement adds in ascending i from +0 (1 + 2^-24 - 1 differs from (1 - 1) + 2^-24 in fp32)"""
    v = np.array([[1.0], [2.0 ** -24], [-1.0], [-0.0]], np.float32)
    out = gn.sequential_segment_sum(v, None, np.array([0, 4, 4]))
    assert out[0, 0] == 0.0 and out[1, 0] == 0.0
    out = gn.sequential_segment_sum(v, np.array([0, 2, 1, 3]), np.array([0, 4]))
    assert out[0, 0] == np.float32(2.0 ** -24)
    neg = gn.sequential_segment_sum(np.array([[-0.0]], np.float32), None, np.array([0, 1]))
    assert np.signbit(neg[0, 0]) == False          # noqa: E712  (+0 + -0 = +0)
