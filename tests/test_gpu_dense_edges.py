"""The non-convolution kernels of a denoising step (csrc/dense.cu) at their edges, against the restatements and the fp32 error
model of tests/dense_numerics.py:
  * farthest point sampling: the selection sequence bit for bit, on all three kernels (k_fps below 8192 points and above the
    cooperative limit, k_fps_coop between, k_fps_cluster for batches), with exact ties across CTAs and register slots;
  * lb2_linear and lb2_head_mlp: every element within the model's bound of fp64, strides, live counts, canaries in every byte the
    kernel must not write, non-finite rows, and the argument checks;
  * lb2_gate_mul and lb2_gather_rows bit-exact against torch on the CPU;
  * the DPM tail's round half to even on exact half-integers;
  * lb2_nn_match_tree (and lb2_nn_match) bit-exact against the brute force at the key-range corners and with live counts."""
import numpy as np
import pytest
import torch

import dense_numerics as dn
import split_numerics as sn
from oracle import me_cpu as ome

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CANARY = -12345.5


@pytest.fixture(scope="module")
def h():
    from lidiff_b200 import _lib
    return _lib.get_handle(DEV)


@pytest.fixture(scope="module")
def coop_limit():
    """most points k_fps_coop takes: 1024 threads x 4 points on every SM"""
    return torch.cuda.get_device_properties(DEV).multi_processor_count * 1024 * 4


@pytest.fixture(scope="module")
def bench_scan():
    from lidiff_b200.synth import range_filter, synthetic_scan
    return torch.tensor(range_filter(synthetic_scan(0)), dtype=torch.float64, device=DEV)


def same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    if a.dtype == torch.float16:
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- farthest point sampling ------------------------------------------------------------------------------------------------
def fps_single(p, ns):
    from lidiff_b200.preprocess import farthest_point_sample
    return farthest_point_sample(p, ns, ordered=False)


def fps_cluster(h, scans, ns):
    """k_fps_cluster directly (no fallback to the single-scan kernel)"""
    pts = torch.cat(scans).contiguous()
    offsets = torch.tensor([0] + [s.shape[0] for s in scans], dtype=torch.int64).cumsum(0).to(DEV)
    idx = torch.full((len(scans), ns), -7, dtype=torch.int32, device=DEV)
    h.farthest_point_sample_batched(pts, offsets, len(scans), max(s.shape[0] for s in scans), ns, idx)
    return idx.long()


def gauss(n, seed, spread=10.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, 3, generator=g, dtype=torch.float64) * spread + offset).to(DEV)


def lattice(nx, ny, nz, seed):
    """a permuted integer lattice: equal distances everywhere, and the first of them in any CTA or register slot"""
    g = torch.Generator().manual_seed(seed)
    p = torch.stack(torch.meshgrid(torch.arange(nx), torch.arange(ny), torch.arange(nz), indexing="ij"), -1).reshape(-1, 3)
    return p[torch.randperm(p.shape[0], generator=g)].double().to(DEV)


def duplicated(n_distinct, copies, seed):
    g = torch.Generator().manual_seed(seed)
    p = (torch.randn(n_distinct, 3, generator=g, dtype=torch.float64) * 5).repeat(copies, 1)
    return p[torch.randperm(p.shape[0], generator=g)].to(DEV)


FPS_CASES = {   # name: (points, n_samples); k_fps below 8192 points, k_fps_coop from 8192 up to the cooperative limit
    "n1": (lambda: gauss(1, 1), 1),
    "n2": (lambda: gauss(2, 2), 2),
    "n8191_all": (lambda: gauss(8191, 3), 8191),
    "n8191_one": (lambda: gauss(8191, 3), 1),
    "n8192_all": (lambda: gauss(8192, 4), 8192),
    "n8192_one": (lambda: gauss(8192, 4), 1),
    "lattice_single_cta": (lambda: lattice(20, 20, 10, 5), 2000),
    "lattice_coop": (lambda: lattice(40, 40, 20, 6), 2000),
    "duplicates_single_cta": (lambda: duplicated(1000, 4, 7), 1500),
    "duplicates_coop": (lambda: duplicated(3000, 4, 8), 3500),
    # above 32 CTAs x 1024 points every lane of the cross-CTA reduction holds several CTAs, and above one slot per thread of the
    # grid every thread holds several points: ties across both
    "lattice_coop_wide": (lambda: lattice(64, 64, 48, 61), 2000),
    "duplicates_coop_wide": (lambda: duplicated(50_000, 4, 62), 2000),
    "identical_single_cta": (lambda: torch.full((100, 3), 3.25, dtype=torch.float64, device=DEV), 50),
    "identical_coop": (lambda: torch.full((10_000, 3), -3.25, dtype=torch.float64, device=DEV), 50),
    "offset_single_cta": (lambda: gauss(5000, 9, offset=1e6), 1000),
    "offset_coop": (lambda: gauss(20_000, 10, offset=1e6), 2000),
}


@pytest.mark.parametrize("case", list(FPS_CASES))
def test_fps_sequence(case):
    make, ns = FPS_CASES[case]
    p = make()
    got = fps_single(p, ns)
    assert torch.equal(got, dn.fps_sequence_torch([p], ns)[0]), case


@pytest.mark.parametrize("extra", [0, 1])
@pytest.mark.parametrize("ns", [1, 300])
def test_fps_at_the_cooperative_limit(coop_limit, extra, ns):
    """n = the limit runs k_fps_coop with every register slot of every CTA live; one more point goes to the single-CTA kernel"""
    p = gauss(coop_limit + extra, 11 + extra)
    assert torch.equal(fps_single(p, ns), dn.fps_sequence_torch([p], ns)[0])


@pytest.mark.parametrize("ns", [1, 18_000])
def test_fps_benchmark_scan(bench_scan, ns):
    assert torch.equal(fps_single(bench_scan, ns), dn.fps_sequence_torch([bench_scan], ns)[0])


def _cluster_size(h):
    return h.fps_batched_capacity() // (1024 * 9)


def test_fps_cluster_full_capacity(h):
    cap = h.fps_batched_capacity()
    assert cap > 0
    scans = [gauss(cap, 21), lattice(30, 30, 30, 22)[: cap // 3]]
    assert torch.equal(fps_cluster(h, scans, 2000), dn.fps_sequence_torch(scans, 2000))


def test_fps_cluster_scans_smaller_than_the_cluster(h):
    """slice = 1 point per CTA (or 2): most CTAs of the small scans own no point"""
    cs = _cluster_size(h)
    for sizes, ns in (([cs - 1, 5, 3, 2], 2), ([1], 1), ([2 * cs - 1, cs + 1, cs], cs)):
        scans = [gauss(n, 30 + n) for n in sizes]
        assert torch.equal(fps_cluster(h, scans, ns), dn.fps_sequence_torch(scans, ns)), sizes


def test_fps_cluster_slice_boundaries(h):
    cs, S = _cluster_size(h), 4000
    sizes = [cs * S, S, S + 1, S - 1, 2 * S, 2 * S + 1, (cs - 1) * S + 1]
    scans = [lattice(20, 20, 10, 40 + i)[:n] if n <= 4000 else gauss(n, 40 + i) for i, n in enumerate(sizes)]
    assert torch.equal(fps_cluster(h, scans, 500), dn.fps_sequence_torch(scans, 500))


def test_fps_cluster_several_waves(h):
    """more scans than clusters fit on the device at once; ties in a duplicated scan"""
    g = torch.Generator().manual_seed(50)
    sizes = torch.randint(3000, 6000, (40,), generator=g).tolist()
    scans = [gauss(n, 51 + i) for i, n in enumerate(sizes)]
    scans[7] = duplicated(1000, 4, 52)
    assert torch.equal(fps_cluster(h, scans, 300), dn.fps_sequence_torch(scans, 300))


# ---- lb2_linear --------------------------------------------------------------------------------------------------------------
def _buf(rows, cols, ld, values, pad):
    """(rows, ld) fp32 device buffer holding `values` (rows, cols) with `pad` in the columns past cols"""
    b = torch.full((rows, ld), pad, dtype=torch.float32)
    b[:, :cols] = values
    return b.to(DEV).contiguous()


LIN_VARIANTS = [  # act, addend, prebias, live count (None: no d_m; else an offset from M, "zero", or "above")
    (0, False, False, None), (1, True, False, "equal"), (2, False, True, "above"), (1, False, True, "below"),
    (2, True, False, "below"), (0, True, True, "zero"),
]


@pytest.mark.parametrize("n_in", [1, 15, 16, 17, 256, 512])
@pytest.mark.parametrize("n_out", [1, 3, 63, 64, 65, 256])
def test_linear_within_the_bound(h, n_in, n_out):
    for M in (1, 63, 64, 65, 5000):
        g = torch.Generator().manual_seed(M * 7 + n_in * 131 + n_out)
        x = torch.randn(M, n_in, generator=g)
        w, b = torch.randn(n_out, n_in, generator=g) * 0.1, torch.randn(n_out, generator=g)
        add, pre = torch.randn(M, n_out, generator=g), torch.randn(n_in, generator=g)
        ldx, ldy, lda = n_in + 3, n_out + 5, n_out + 2
        dx = _buf(M, n_in, ldx, x, float("nan"))                 # a read of the padding would poison the row
        da = _buf(M, n_out, lda, add, float("nan"))
        dw, db, dpre = w.to(DEV), b.to(DEV), pre.to(DEV)
        for act, use_add, use_pre, live in LIN_VARIANTS:
            m_live = {None: M, "equal": M, "above": M, "below": M - 1, "zero": 0}[live]
            d_m = None if live is None else torch.tensor([{"above": M + 10}.get(live, m_live)], dtype=torch.int32, device=DEV)
            y = torch.full((M, ldy), CANARY, device=DEV)
            h.linear(dx, ldx, dw, db, da if use_add else None, lda, M, d_m, n_in, n_out, act, y, ldy,
                     dpre if use_pre else None, 1)
            ref, bound = dn.linear_reference(x[:m_live].numpy(), w.numpy(), b.numpy(), add[:m_live].numpy() if use_add else None,
                                             act, pre.numpy() if use_pre else None, 1)
            y = y.cpu()
            what = (M, act, use_add, use_pre, live)
            assert dn.within(y[:m_live, :n_out].numpy(), ref, bound) <= 1.0, what
            canary = torch.full_like(y, CANARY)
            assert same_bits(y[m_live:], canary[m_live:]), ("rows past the live count written",) + what
            assert same_bits(y[:, n_out:], canary[:, n_out:]), ("padding columns written",) + what


def test_linear_nan_row_stays_in_its_row(h):
    M, n_in, n_out = 5000, 17, 65
    g = torch.Generator().manual_seed(3)
    x, w, b = torch.randn(M, n_in, generator=g), torch.randn(n_out, n_in, generator=g) * 0.1, torch.randn(n_out, generator=g)
    x[1234, 5] = float("nan")
    y = torch.full((M, n_out), CANARY, device=DEV)
    h.linear(x.to(DEV), n_in, w.to(DEV), b.to(DEV), None, 0, M, None, n_in, n_out, 1, y, n_out)
    y = y.cpu()
    assert torch.isnan(y[1234]).all()
    rest = torch.ones(M, dtype=torch.bool)
    rest[1234] = False
    ref, bound = dn.linear_reference(x[rest].numpy(), w.numpy(), b.numpy(), act=1)
    assert dn.within(y[rest].numpy(), ref, bound) <= 1.0


# ---- lb2_head_mlp ------------------------------------------------------------------------------------------------------------
def _head(h, n_in, n_hid, n_out, act, npass, M, m_live, seed, pad=4):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(npass, M, n_in, generator=g)
    w0, b0 = torch.randn(n_hid, n_in, generator=g) / 10, torch.randn(n_hid, generator=g)
    w1, b1 = torch.randn(n_out, n_hid, generator=g) / 4, torch.randn(n_out, generator=g)
    ldx, ldy = n_in + pad, n_out + 3
    dx = torch.full((npass, M, ldx), float("nan"))
    dx[..., :n_in] = x
    dx = dx.to(DEV)
    y = torch.full((npass, M, ldy), CANARY, device=DEV)
    d_m = None if m_live == M else torch.tensor([m_live], dtype=torch.int32, device=DEV)
    h.head_mlp(dx, ldx, M * ldx, *(t.to(DEV) for t in (w0, b0, w1, b1)), M, d_m, n_in, n_hid, n_out, act, npass, y, ldy, M * ldy)
    y = y.cpu()
    canary = torch.full_like(y, CANARY)
    for p in range(npass):
        ref, bound = dn.head_mlp_reference(x[p, :m_live].numpy(), w0.numpy(), b0.numpy(), w1.numpy(), b1.numpy(), act)
        what = (n_in, n_hid, n_out, act, npass, M, m_live, p)
        assert dn.within(y[p, :m_live, :n_out].numpy(), ref, bound) <= 1.0, what
        assert same_bits(y[p, m_live:], canary[p, m_live:]), ("rows past the live count written",) + what
        assert same_bits(y[p, :, n_out:], canary[p, :, n_out:]), ("padding columns written",) + what


@pytest.mark.parametrize("n_in", list(range(16, 129, 16)))
@pytest.mark.parametrize("n_hid", [1, 20, 64])
def test_head_mlp_shapes(h, n_in, n_hid):
    for i, n_out in enumerate([1, 3, 4, 5, 18, 24]):
        for M, m_live in ((1, 1), (7, 7), (8, 8), (9, 9), (300, 201)):
            _head(h, n_in, n_hid, n_out, (0, 2)[i % 2], 1 + (M + i) % 2, M, m_live, n_in * 1000 + n_hid * 10 + n_out + M)


@pytest.mark.parametrize("shape", [(96, 20, 3, 0), (96, 20, 18, 2), (128, 64, 24, 2), (16, 1, 1, 0)])
def test_head_mlp_grid_sweeps(h, shape):
    """the grid is capped at num_sms x 8 CTAs of 64 rows: one sweep -1, one sweep, one sweep +1 and the engine's 180 000 rows"""
    sweep = torch.cuda.get_device_properties(DEV).multi_processor_count * 8 * 64
    n_in, n_hid, n_out, act = shape
    for M, m_live in ((sweep - 1, sweep - 1), (sweep, sweep), (sweep + 1, sweep + 1), (180_000, 179_995), (sweep + 64, sweep + 1)):
        _head(h, n_in, n_hid, n_out, act, 2, M, m_live, M + n_out)


def test_head_mlp_and_linear_refuse_bad_arguments(h):
    """shape checks, an x that is not 16-byte aligned, a pass stride that is not a multiple of 4 floats, a short ld_addend"""
    M = 64
    x = torch.randn(2 * M * 128 + 4, device=DEV)
    w0, b0, w1, b1 = torch.randn(64 * 136, device=DEV), torch.randn(65, device=DEV), torch.randn(25 * 65, device=DEV), torch.randn(25, device=DEV)
    y = torch.full((2, M, 32), CANARY, device=DEV)

    def head(xp, ldx, xps, n_in, n_hid, n_out, npass=1):
        h.head_mlp(xp, ldx, xps, w0, b0, w1, b1, M, None, n_in, n_hid, n_out, 0, npass, y, 32, M * 32)

    head(x, 96, M * 96, 96, 20, 3, 2)                             # the valid call these variants break
    for args in ((x, 8, 0, 8, 20, 3), (x, 136, 0, 136, 20, 3), (x, 100, 0, 100, 20, 3), (x, 96, 0, 96, 65, 3), (x, 96, 0, 96, 20, 25),
                 (x[1:], 96, 0, 96, 20, 3), (x[2:], 96, 0, 96, 20, 3), (x, 96, M * 96 + 1, 96, 20, 3, 2), (x, 96, M * 96 + 2, 96, 20, 3, 2)):
        with pytest.raises(RuntimeError, match="lb2_head_mlp"):
            head(*args)
    torch.cuda.synchronize()
    yl = torch.full((M, 8), CANARY, device=DEV)
    add = torch.randn(M, 8, device=DEV)
    with pytest.raises(RuntimeError, match="ld_addend"):
        h.linear(x, 16, w0, b0, add, 7, M, None, 16, 8, 0, yl, 8)
    h.linear(x, 16, w0, b0, add, 8, M, None, 16, 8, 0, yl, 8)
    torch.cuda.synchronize()


# ---- lb2_gate_mul / lb2_gather_rows ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [18, 32])
@pytest.mark.parametrize("with_idx", [True, False])
@pytest.mark.parametrize("outs", ["both", "out", "out_h"])
def test_gate_mul_bit_exact(h, c, with_idx, outs):
    cap, live = 3000, 2345
    g = torch.Generator().manual_seed(c + 2 * with_idx)
    x, table = torch.randn(cap, c, generator=g) * 3, torch.randn(50, c, generator=g)
    idx = torch.randint(0, 50, (cap,), generator=g, dtype=torch.int32)
    ref = x * (table[idx.long()] if with_idx else table[0:1])
    for d_m in (None, live):
        m = cap if d_m is None else live
        out = torch.full((cap, c), CANARY, device=DEV) if outs != "out_h" else None
        out_h = torch.full((cap, 2 * c), -7.0, dtype=torch.float16, device=DEV) if outs != "out" else None
        dm = None if d_m is None else torch.tensor([d_m], dtype=torch.int32, device=DEV)
        h.gate_mul(x.to(DEV), table.to(DEV), idx.to(DEV) if with_idx else None, dm, cap, c, out, out_h)
        if out is not None:
            out = out.cpu()
            assert same_bits(out[:m], ref[:m])
            assert same_bits(out[m:], torch.full_like(out[m:], CANARY)), "rows past the live count written"
        if out_h is not None:
            out_h = out_h.cpu()
            hi, lo = sn.split(ref[:m])
            assert same_bits(out_h[:m, :c], hi) and same_bits(out_h[:m, c:], lo)
            assert same_bits(out_h[m:], torch.full_like(out_h[m:], -7.0)), "rows past the live count written"


@pytest.mark.parametrize("c", [3, 18, 32])
def test_gather_rows_bit_exact(h, c):
    g = torch.Generator().manual_seed(c)
    src = torch.randn(777, c, generator=g)
    n = 5000
    idx = torch.randint(0, 777, (n,), generator=g, dtype=torch.int32)
    idx[:3] = torch.tensor([0, 776, 0], dtype=torch.int32)
    out = torch.full((n + 100, c), CANARY, device=DEV)
    h.gather_rows(src.to(DEV), idx.to(DEV), n, c, out)
    out = out.cpu()
    assert same_bits(out[:n], src[idx.long()])
    assert same_bits(out[n:], torch.full_like(out[n:], CANARY))


# ---- the DPM tail: round half to even -------------------------------------------------------------------------------------------
def half_integer_inputs(div_mode, res=0.05):
    """fp32 x whose x / res (div_mode 0) or x * float32(1 / res) (div_mode 1) is exactly k + 1/2, for k of both signs and parities"""
    r = np.float32(res)
    inv = np.float32(1) / r
    xs, ks = [], []
    for k in list(range(-1003, -995)) + list(range(-4, 4)) + list(range(995, 1003)):
        x = np.float32((k + 0.5) * res)
        for _ in range(20):
            x = np.nextafter(x, np.float32(-np.inf))
        for _ in range(40):
            if (x / r if div_mode == 0 else x * inv) == np.float32(k + 0.5):
                xs.append(x)
                ks.append(k)
                break
            x = np.nextafter(x, np.float32(np.inf))
    return np.array(xs, np.float32), np.array(ks)


@pytest.mark.parametrize("div_mode", [0, 1])
@pytest.mark.parametrize("second", [0, 1])
def test_dpm_tail_rounds_half_to_even(h, div_mode, second):
    """zero eps, noise and sample: x_next is x_init, and its coordinate k + 1/2 must round to the even neighbour"""
    from lidiff_b200._lib import DpmCoef
    from lidiff_b200.scheduler import DPMSolverMultistepScheduler as S
    xs, ks = half_integer_inputs(div_mode)
    assert (ks < 0).sum() >= 10 and (ks > 0).sum() >= 10 and (ks % 2 == 0).sum() >= 10 and (ks % 2 == 1).sum() >= 10
    x = torch.from_numpy(np.stack([xs, xs[::-1], np.roll(xs, 5)], 1).copy())
    n = x.shape[0]
    s = S(1000, 3.5e-5, 0.007, "linear", algorithm_type="sde-dpmsolver++", solver_order=2)
    s.set_timesteps(50)
    c = s.coefficients(7)
    cf = DpmCoef(c["c_sample"], c["c_x0"], c["c_noise"], c["sigma_s"], c["alpha_s"], c["inv_r0"] if second else 0.0,
                 6.0, 0.05, second, div_mode, 1)
    z = torch.zeros(n, 3, device=DEV)
    x_next = torch.empty(n, 3, device=DEV)
    coord = torch.full((n, 4), CANARY, device=DEV)
    bcol = torch.arange(n, dtype=torch.float32, device=DEV) % 4
    h.guidance_dpm_step(z, z, None, x.to(DEV), x.double().to(DEV), z, torch.zeros(n, 3, dtype=torch.float64, device=DEV), n, cf,
                        None, x_next, coord, bcol)
    coord = coord.cpu()
    assert same_bits(x_next.cpu(), x)
    expect = torch.from_numpy(np.where(ks % 2 == 0, ks, ks + 1).astype(np.float32))
    assert torch.equal(coord[:, 1], expect), "k + 1/2 must round to the even neighbour"
    assert torch.equal(coord[:, 1:], ome.quantize(x, 0.05, "div" if div_mode == 0 else "mul"))
    assert torch.equal(coord[:, 0], bcol.cpu())


# ---- lb2_nn_match_tree -------------------------------------------------------------------------------------------------------
LO, HI = -131072, 131071


def _corner_sets(seed):
    g = torch.Generator().manual_seed(seed)
    ax = torch.tensor([LO, LO + 1, -1, 0, 1, HI - 1, HI])
    corners = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    keys = torch.cat([corners, torch.randint(LO, HI + 1, (2000, 3), generator=g)])
    kb = torch.where(torch.rand(keys.shape[0], generator=g) < 0.5, 0, 1023)
    keys = torch.cat([kb[:, None], keys], 1)
    keys = torch.cat([keys, keys[:300]])                                    # duplicated keys: the lower row wins
    q = torch.cat([corners, torch.randint(LO, HI + 1, (20_000, 3), generator=g), keys[:500, 1:] + torch.randint(-2, 3, (500, 3), generator=g)])
    q = q.clamp(LO, HI)
    qb = torch.tensor([0, 1023, 512])[torch.randint(0, 3, (q.shape[0],), generator=g)]  # batch 512 has no key
    return torch.cat([qb[:, None], q], 1).int(), keys.int()


def test_nn_match_tree_key_range_corners_and_live_counts(h):
    q, k = _corner_sets(1)
    ref = torch.from_numpy(dn.nn_brute(q.numpy(), k.numpy()))
    nq, nk = q.shape[0], k.shape[0]
    qd = torch.cat([q, torch.full((77, 4), 5, dtype=torch.int32)]).to(DEV).contiguous()       # capacity above the live count
    kd = torch.cat([k, torch.zeros(33, 4, dtype=torch.int32)]).to(DEV).contiguous()           # a live key at (0,0,0,0) would win ties
    d_nq = torch.tensor([nq], dtype=torch.int32, device=DEV)
    d_nk = torch.tensor([nk], dtype=torch.int32, device=DEV)
    tree = h.nn_tree(kd, d_nk, nk + 33)
    g = torch.Generator().manual_seed(2)
    hint = torch.randint(0, nk, (999,), generator=g).int().to(DEV)
    hof = torch.randint(0, 999, (nq + 77,), generator=g).int().to(DEV)
    for hinted in (False, True):
        idx = torch.full((nq + 77,), -5, dtype=torch.int32, device=DEV)
        if hinted:
            h.nn_match_tree(qd, d_nq, nq + 77, tree, nk + 33, idx, kd, hof, hint)
        else:
            h.nn_match_tree(qd, d_nq, nq + 77, tree, nk + 33, idx)
        idx = idx.cpu()
        assert torch.equal(idx[:nq].long(), ref), ("hinted" if hinted else "plain")
        assert (idx[nq:] == -5).all(), "rows past the live count written"
    a = torch.full((nq + 77,), -5, dtype=torch.int32, device=DEV)
    h.nn_match(qd, d_nq, nq + 77, kd, d_nk, nk + 33, 0, a)
    a = a.cpu()
    assert torch.equal(a[:nq].long(), ref) and (a[nq:] == -5).all(), "brute-force kernel"
