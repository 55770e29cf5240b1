"""GPU parity tests, kernel by kernel: the CUDA library (through its C ABI) against the CPU oracle on
identical seeded inputs.  Integer / index results bit-exact, floating point within the tolerance
stated at each assert (north star: 1e-3 relative fp32)."""
import numpy as np
import pytest
import torch

from oracle import me_cpu as ome
from oracle.dpm import DPMSolverSDE2M
from oracle.pipeline import farthest_point_sample as fps_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def H():
    from lidiff_b200 import _lib
    return _lib.get_handle(DEV)


def rel_err(a, b):
    """per-element |a-b| / (|b| + rms(b)) as in SURVEY.md 8c-iii"""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs() / (b.abs() + b.pow(2).mean().sqrt() + 1e-30)).max().item()


def random_field(n, spread, seed, batch=1):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(n, 3, generator=g) * spread
    b = torch.sort(torch.randint(0, batch, (n, 1), generator=g).float(), dim=0).values
    coords = torch.cat([b, torch.round(pts / 0.05)], 1)
    return pts, coords


# ---------------------------------------------------------------------------------------------------------
def test_torch_cuda_scalar_division_is_reciprocal_multiply():
    """pins which quantisation form the reference's own CUDA path computes (SURVEY.md App. B.6)"""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2_000_000, generator=g) * 30
    ref_gpu = torch.round(x.to(DEV) / 0.05).cpu()
    mul = ome.quantize(x, 0.05, "mul")
    div = ome.quantize(x, 0.05, "div")
    n_mul, n_div = int((ref_gpu != mul).sum()), int((ref_gpu != div).sum())
    print(f"torch CUDA round(x/0.05): differs from x*20f in {n_mul}, from true division in {n_div} of {x.numel()}")
    assert n_mul == 0, "engine div_mode=1 would not match torch's CUDA lowering"


@pytest.mark.parametrize("mode", [0, 1])
def test_quantize_bit_exact(mode):
    g = torch.Generator().manual_seed(1)
    x = torch.cat([torch.randn(500_000, generator=g) * 30, torch.tensor([0.025, 0.075, 0.125, -0.025, -0.075, 0.0])])
    out = torch.empty_like(x, device=DEV)
    H().quantize(x.to(DEV), 0.05, mode, out)
    assert torch.equal(out.cpu(), ome.quantize(x, 0.05, "div" if mode == 0 else "mul"))


@pytest.mark.parametrize("n,spread,batch", [(50_000, 2.0, 1), (20_000, 0.2, 3), (7, 1.0, 1), (4096, 0.0, 1)])
def test_voxelise_and_levels_bit_exact(n, spread, batch):
    from lidiff_b200 import me
    pts, coords = random_field(n, spread, n, batch)
    of = ome.TensorField(pts, coords)
    os_ = of.sparse()
    f = me.TensorField(pts.to(DEV), coords.to(DEV))
    s = f.sparse()
    assert torch.equal(s.C.cpu(), os_.C), "level-0 rows / order"
    assert torch.equal(f.inverse_mapping.cpu(), torch.from_numpy(os_.geom.inverse)), "inverse map"
    assert rel_err(s.F, os_.F) < 1e-5
    cm = s.coordinate_manager
    for ts in (2, 4, 8, 16):
        assert torch.equal(cm.level(ts).C.cpu(), torch.from_numpy(os_.geom.stride_level(ts))), f"stride {ts} rows"
        assert torch.equal(cm.level(ts).parent_inverse[:cm.level(ts // 2).n].long().cpu(),
                           torch.from_numpy(os_.geom.fine2coarse[ts])), f"fine->coarse {ts}"


def _pairs_from_nbr(nbr):
    nbr = nbr.cpu().numpy()
    out = []
    for k in range(nbr.shape[0]):
        o = np.nonzero(nbr[k] >= 0)[0]
        out.append(set(zip(nbr[k][o].tolist(), o.tolist())))
    return out


@pytest.mark.parametrize("spread", [1.0, 0.1])
def test_kernel_maps_equal_oracle_pair_sets(spread):
    from lidiff_b200 import me
    pts, coords = random_field(30_000, spread, 5)
    og = ome.TensorField(pts, coords).sparse().geom
    cm = me.TensorField(pts.to(DEV), coords.to(DEV)).sparse().coordinate_manager
    for ts in (1, 2, 4):
        for (ks, stride, tr) in ((3, 1, False), (2, 2, False)):
            got = _pairs_from_nbr(cm.kernel_map(ts, ks, stride, tr))
            ref = [set(zip(i.tolist(), o.tolist())) for (i, o) in og.kernel_map(ts, ks, stride, tr)]
            assert got == ref, (ts, ks, stride)
        got = _pairs_from_nbr(cm.kernel_map(ts * 2, 2, 2, True))
        ref = [set(zip(i.tolist(), o.tolist())) for (i, o) in og.kernel_map(ts * 2, 2, 2, True)]
        assert got == ref, (ts, "transposed")


CONV_CASES = [  # cin, cout, ks, stride, transposed
    (3, 32, 3, 1, False), (32, 32, 3, 1, False), (32, 64, 2, 2, False), (64, 48, 2, 2, True),
    (96, 96, 3, 1, False), (128, 256, 1, 1, False), (20, 7, 3, 1, False),
    (64, 64, 2, 2, True), (256, 256, 3, 1, False), (128, 128, 3, 1, False), (256, 128, 2, 2, True), (48, 32, 3, 1, False),
]


def tc_supported(cin, cout):
    return cin % 16 == 0 and cout % 32 == 0 and 32 <= cout <= 256


@pytest.mark.parametrize("cin,cout,ks,stride,tr", CONV_CASES)
@pytest.mark.parametrize("algo", [1, 2])
def test_sparse_conv_matches_oracle(cin, cout, ks, stride, tr, algo):
    from lidiff_b200 import me
    if algo == 2 and not tc_supported(cin, cout):
        pytest.skip("shape not taken by the tensor-core variant")
    pts, coords = random_field(12_000, 0.3, 11)
    g = torch.Generator().manual_seed(cin * 131 + cout)
    of = ome.TensorField(pts, coords).sparse()
    f = me.TensorField(pts.to(DEV), coords.to(DEV)).sparse()
    ts_in = 2 if tr else 1
    Min = of.geom.stride_level(ts_in).shape[0]
    Fin = torch.randn(Min, cin, generator=g)
    if ks == 1:
        layer = me.MinkowskiConvolution(cin, cout, kernel_size=1, stride=1, dimension=3)
    elif tr:
        layer = me.MinkowskiConvolutionTranspose(cin, cout, kernel_size=ks, stride=stride, dimension=3)
    else:
        layer = me.MinkowskiConvolution(cin, cout, kernel_size=ks, stride=stride, dimension=3)
    layer.algo = algo
    W = torch.randn(layer.kernel.shape, generator=g) / np.sqrt(cin * ks ** 3)
    layer.kernel.data = W.clone()
    layer = layer.to(DEV)
    xin = me.SparseTensor(Fin.to(DEV), coordinate_manager=f.coordinate_manager, tensor_stride=ts_in)
    y = layer(xin)
    oy = ome.conv(ome.SparseTensor(Fin.double(), of.geom, ts_in), W.double(), ks, stride, tr)
    assert y.F.shape == oy.F.shape
    e = rel_err(y.F, oy.F)
    print(f"conv {cin}->{cout} ks{ks} s{stride} tr{tr} algo{algo}: rel err {e:.3e}")
    assert e < (1e-4 if algo == 1 else 5e-5), "conv vs fp64 oracle (fp32 FFMA / FP16x3 two-level tensor core)"


@pytest.mark.parametrize("algo,c1,c2,cout", [(1, 32, 16, 24), (2, 32, 16, 64), (2, 96, 32, 96), (2, 256, 128, 256)])
def test_sparse_conv_fused_epilogue_two_passes_and_concat(algo, c1, c2, cout):
    """BN affine + residual + ReLU + gate + two K segments + two guidance passes in one launch"""
    from lidiff_b200 import _lib, me
    from lidiff_b200._lib import ConvDesc, ConvIO
    pts, coords = random_field(9_000, 0.2, 21)
    g = torch.Generator().manual_seed(5)
    of = ome.TensorField(pts, coords).sparse()
    f = me.TensorField(pts.to(DEV), coords.to(DEV)).sparse()
    cm = f.coordinate_manager
    M = of.F.shape[0]
    A = torch.randn(2, M, c1, generator=g)
    B = torch.randn(1, M, c2, generator=g)
    R = torch.randn(2, M, cout, generator=g)
    W = torch.randn(27, c1 + c2, cout, generator=g) * 0.05
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g)
    table = torch.randn(50, cout, generator=g)
    gidx = torch.randint(0, 50, (M,), generator=g, dtype=torch.int32)
    dev = lambda t: t.to(DEV).contiguous()
    dA, dB, dR, dW, dS, dT, dTab, dG = map(dev, (A, B, R, W, scale, shift, table, gidx))
    out = torch.zeros(2, M, cout, device=DEV)
    outg = torch.zeros(2, M, cout, device=DEV)
    nbr = cm.kernel_map(1, 3, 1, False)
    d_m = torch.tensor([M], dtype=torch.int32, device=DEV)
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, 27
    d.weight, d.scale, d.shift, d.relu = dW.data_ptr(), dS.data_ptr(), dT.data_ptr(), 1
    packed = H().pack_weights(dW) if algo == 2 else None
    d.weight_packed = packed.data_ptr() if packed is not None else None
    d.nbr, d.nbr_stride, d.d_mout, d.mout_cap, d.npass = nbr.data_ptr(), nbr.stride(0), d_m.data_ptr(), M, 2
    d.io[0] = ConvIO(dA[0].data_ptr(), dB[0].data_ptr(), dR[0].data_ptr(), out[0].data_ptr(), dTab.data_ptr(), dG.data_ptr(), outg[0].data_ptr())
    d.io[1] = ConvIO(dA[1].data_ptr(), dB[0].data_ptr(), dR[1].data_ptr(), out[1].data_ptr(), dTab.data_ptr(), None, outg[1].data_ptr())
    H().spconv(d, algo)
    tol = 1e-4 if algo == 1 else 5e-5
    for p in range(2):
        xin = ome.SparseTensor(torch.cat([A[p], B[0]], 1).double(), of.geom, 1)
        y = ome.conv(xin, W.double(), 3).F * scale.double() + shift.double() + R[p].double()
        y = torch.relu(y)
        e = rel_err(out[p], y)
        print(f"fused conv algo{algo} {c1}+{c2}->{cout} pass {p}: rel err {e:.3e}")
        assert e < tol
        gate = table[gidx.long()] if p == 0 else table[0:1]
        assert rel_err(outg[p], y * gate.double()) < tol


def test_nn_match_bit_exact_with_ties():
    g = torch.Generator().manual_seed(3)
    q = torch.cat([torch.zeros(40_000, 1), torch.randint(-60, 60, (40_000, 3), generator=g).float() * 2], 1)
    k = torch.cat([torch.zeros(3_000, 1), torch.randint(-8, 8, (3_000, 3), generator=g).float() * 16], 1)   # many duplicates/ties
    ref = ome.match_part_to_full(q.int(), k.int())
    idx = torch.empty(q.shape[0], dtype=torch.int32, device=DEV)
    H().nn_match(q.int().to(DEV), None, q.shape[0], k.int().to(DEV), None, k.shape[0], 0, idx)
    assert torch.equal(idx.long().cpu(), ref)
    # the reference's own expression through the keops surface, two batches
    from lidiff_b200.keops import LazyTensor
    q2, k2 = q.clone(), k.clone()
    q2[20_000:, 0], k2[1_500:, 0] = 1, 1
    ref2 = ome.match_part_to_full(q2.int(), k2.int())
    fc, pc = q2.to(DEV), k2.to(DEV)
    s = fc.max() * 2.0
    fc[:, 0] *= s
    pc[:, 0] *= s
    got = ((LazyTensor(fc[:, None, :]) - LazyTensor(pc[None, :, :])) ** 2).sum(-1).argKmin(1, dim=1)[:, 0]
    assert torch.equal(got.cpu(), ref2)


@pytest.mark.parametrize("m,n_in,n_out,act", [(5000, 256, 256, 1), (777, 96, 20, 1), (777, 20, 3, 0), (1, 512, 96, 0), (300, 20, 18, 2)])
def test_linear_matches_torch(m, n_in, n_out, act):
    g = torch.Generator().manual_seed(m + n_out)
    x, w, b = torch.randn(m, n_in, generator=g), torch.randn(n_out, n_in, generator=g) * 0.1, torch.randn(n_out, generator=g)
    y = torch.empty(m, n_out, device=DEV)
    H().linear(x.to(DEV), n_in, w.to(DEV), b.to(DEV), None, 0, m, None, n_in, n_out, act, y, n_out)
    ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
    ref = torch.nn.functional.leaky_relu(ref, 0.1) if act == 1 else (torch.tanh(ref) if act == 2 else ref)
    assert rel_err(y, ref) < 1e-5
    # hoisted-gate form: W2 . leaky(x + prebias) + b
    pre = torch.randn(n_in, generator=g)
    H().linear(x.to(DEV), n_in, w.to(DEV), b.to(DEV), None, 0, m, None, n_in, n_out, 0, y, n_out, pre.to(DEV), 1)
    ref = torch.nn.functional.linear(torch.nn.functional.leaky_relu(x.double() + pre.double(), 0.1), w.double(), b.double())
    assert rel_err(y, ref) < 1e-5


@pytest.mark.parametrize("second,T,i,div_mode,with_eps,batch", [
    pytest.param(0, 50, 0, 1, True, False, id="0"), pytest.param(1, 50, 7, 1, True, False, id="1"),
    pytest.param(1, 50, 7, 0, True, False, id="div_mode0"),
    pytest.param(1, 50, 7, 1, False, True, id="no_eps_out-batch_col"),         # the engine's loop: eps_out None, a batch engine's column
    pytest.param(1, 50, 49, 1, False, True, id="last_step_T50"),               # second order
    pytest.param(1, 10, 9, 0, False, False, id="last_step_T10"),               # lower_order_final: first order although x0 is stored
])
def test_guidance_dpm_step_bit_exact(second, T, i, div_mode, with_eps, batch):
    """given identical eps the fused tail reproduces torch's fp64 evaluation bit for bit (x_next AND coords).  `second`: an x0
    prediction is stored; the update is second order unless it is the last step of fewer than 15 (engine.step's rule)"""
    from lidiff_b200._lib import DpmCoef
    from lidiff_b200.scheduler import DPMSolverMultistepScheduler as S
    n, m = 60_000, 20_000
    g = torch.Generator().manual_seed(9 + second + 100 * (T != 50 or i not in (0, 7)) + 10 * (1 - div_mode) + 20 * batch)
    inv = torch.randint(0, m, (n,), generator=g)
    e_c, e_u = torch.randn(m, 3, generator=g), torch.randn(m, 3, generator=g)
    x_init = torch.randn(1, n, 3, generator=g, dtype=torch.float64) * 20
    x_t = (x_init + torch.randn(1, n, 3, generator=g, dtype=torch.float64)).float()
    noise = torch.randn(1, n, 3, generator=g)
    x0_prev = torch.randn(1, n, 3, generator=g, dtype=torch.float64)
    bcol = torch.randint(0, 4, (n,), generator=g).float() if batch else None
    o = DPMSolverSDE2M()
    o.set_timesteps(T)
    if second:
        o.model_outputs = [None, x0_prev.clone()]
        o.lower_order_nums = 1
    eps = (e_u + 6.0 * (e_c - e_u))[inv][None]
    sample = x_t - x_init
    x_next_ref = (x_init + o.step(eps, o.timesteps[i], sample, noise[0][None])).float()
    coord_ref = ome.quantize(x_next_ref, 0.05, "div" if div_mode == 0 else "mul")
    s = S(1000, 3.5e-5, 0.007, "linear", algorithm_type="sde-dpmsolver++", solver_order=2)
    s.set_timesteps(T)
    c = s.coefficients(i)
    so = int(second and not (i == T - 1 and T < 15))
    cf = DpmCoef(c["c_sample"], c["c_x0"], c["c_noise"], c["sigma_s"], c["alpha_s"], c.get("inv_r0", 0.0) if so else 0.0,
                 6.0, 0.05, so, div_mode, 1)
    d = lambda t: t.to(DEV).contiguous()
    x0s = d(x0_prev[0])
    x_next = torch.empty(n, 3, device=DEV)
    coord = torch.empty(n, 4, device=DEV)
    eps_out = torch.empty(n, 3, device=DEV) if with_eps else None
    H().guidance_dpm_step(d(e_c), d(e_u), d(inv.int()), d(x_t[0]), d(x_init[0]), d(noise[0]), x0s, n, cf, eps_out, x_next, coord,
                          d(bcol) if batch else None)
    if with_eps:
        assert torch.equal(eps_out.cpu(), eps[0]), "guidance"
    assert torch.equal(x_next.cpu(), x_next_ref[0]), "x_next"
    assert torch.equal(coord[:, 1:].cpu(), coord_ref[0]), "next coordinates"
    assert torch.equal(coord[:, 0].cpu(), bcol if batch else torch.zeros(n)), "batch column"
    assert torch.equal(x0s.cpu(), o.model_outputs[-1][0]), "multistep state"


def test_farthest_point_sampling_bit_exact():
    from lidiff_b200.preprocess import farthest_point_sample
    g = np.random.default_rng(0)
    p = g.normal(size=(20_000, 3)) * 10
    ref = fps_oracle(p, 500)
    got = farthest_point_sample(torch.tensor(p, device=DEV), 500).cpu().numpy()
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("n_out,out_act,npass", [(3, 0, 2), (18, 2, 1)])
def test_head_mlp_matches_torch(n_out, out_act, npass):
    """lb2_head_mlp: Linear(96,20) + LeakyReLU(0.1) + Linear(20,n_out) (+ tanh) per row, rows from a device count, both passes in one launch"""
    h = H()
    g = torch.Generator().manual_seed(3)
    cap, m = 5000, 4321
    x = torch.randn(npass, cap, 96, generator=g)
    w0, b0 = torch.randn(20, 96, generator=g) / 10, torch.randn(20, generator=g)
    w1, b1 = torch.randn(n_out, 20, generator=g) / 4, torch.randn(n_out, generator=g)
    dx, dw0, db0, dw1, db1 = (t.to(DEV).contiguous() for t in (x, w0, b0, w1, b1))
    y = torch.full((npass, cap, n_out), 7.0, device=DEV)
    d_m = torch.tensor([m], dtype=torch.int32, device=DEV)
    h.head_mlp(dx, 96, cap * 96, dw0, db0, dw1, db1, cap, d_m, 96, 20, n_out, out_act, npass, y, n_out, cap * n_out)
    torch.cuda.synchronize()
    ref = torch.nn.functional.leaky_relu(x[:, :m].double() @ w0.double().t() + b0.double(), 0.1) @ w1.double().t() + b1.double()
    if out_act == 2:
        ref = torch.tanh(ref)
    assert (y[:, :m].double().cpu() - ref).abs().max().item() < 2e-5
    assert (y[:, m:] == 7.0).all(), "rows beyond the live count must stay untouched"


@pytest.mark.parametrize("spread,live", [(0.3, 1.0), (1.5, 0.6)])
def test_kernel_map_self_equals_the_generic_map(spread, live):
    """lb2_kernel_map_self (13 probes + mirrored writes) builds the table, row masks and pair count of lb2_kernel_map(ks=3) bit for bit,
    also when fewer rows are live than the capacity"""
    h = H()
    pts, coords = random_field(40_000, spread, 11)
    N = coords.shape[0]
    from lidiff_b200.engine import Geometry
    g = Geometry(h, N)
    g.build(coords.to(DEV).contiguous(), N)
    for lvl in (0, 2, 4):
        M = g.sizes()[lvl]
        C, d_n = g.C[lvl], g.d_n[lvl]
        if live < 1.0:                                  # a grid over the first rows only: fewer live rows than the capacity
            d_in = torch.tensor([max(1, int(M * live))], dtype=torch.int32, device=DEV)
            C, d_n = torch.zeros_like(g.C[lvl]), torch.zeros(1, dtype=torch.int32, device=DEV)
            h.unique_build(None, g.C[lvl], d_in, N, 1 << lvl, g.grid[lvl], C, torch.zeros_like(g.inv[lvl]), d_n, g.scratch)
        a, b = torch.full((27, N), 5, dtype=torch.int32, device=DEV), torch.full((27, N), 6, dtype=torch.int32, device=DEV)
        ma, mb = torch.full((N,), 9, dtype=torch.int32, device=DEV), torch.full((N,), 8, dtype=torch.int32, device=DEV)
        pa, pb = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
        h.kernel_map(g.grid[lvl], C, d_n, N, 3, 1 << lvl, a, N, pa, ma)
        h.kernel_map_self(g.grid[lvl], C, d_n, N, 1 << lvl, b, N, pb, mb)
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(ma, mb) and int(pa) == int(pb) and int(pa) >= int(d_n)


def test_tile_order_sorts_tiles_by_the_offsets_they_run():
    """lb2_tile_order: order128 / order256 are permutations of the live tiles of the row order, by descending popcount of the OR of
    the tile's row masks; entries beyond the live tiles are -1"""
    from lidiff_b200.engine import Geometry
    h = H()
    pts, coords = random_field(50_000, 0.5, 23)
    N = coords.shape[0]
    g = Geometry(h, N)
    g.build(coords.to(DEV).contiguous(), N)
    sizes = g.sizes()
    for nbr, perm, lvl in ((g.nbr3[1], g.perm3[1], 1), (g.nbr3[3], g.perm3[3], 3), (g.nbr_dn[2], g.perm_dn[2], 2)):
        M = sizes[lvl]
        mask = g.mask_of[nbr.data_ptr()][:M].cpu().numpy().astype(np.uint32)
        pm = mask[perm[:M].cpu().numpy()]
        o128, o256 = (t.cpu().numpy() for t in g.tile_order_of[nbr.data_ptr()])
        for T, order in ((128, o128), (256, o256)):
            nt = (M + T - 1) // T
            cost = np.array([bin(int(np.bitwise_or.reduce(pm[t * T:(t + 1) * T]))).count("1") for t in range(nt)])
            assert np.array_equal(np.sort(order[:nt]), np.arange(nt)), "not a permutation of the live tiles"
            assert (order[nt:] == -1).all()
            assert (np.diff(cost[order[:nt]]) <= 0).all(), "tiles must come out by descending cost"


@pytest.mark.parametrize("spread,algo", [(1.0, 1), (0.1, 2), (1.0, 2)])
def test_row_order_is_a_permutation_and_does_not_change_results(spread, algo):
    """lb2_row_order only reschedules tiles: perm is a permutation grouped by mask class, conv output identical"""
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    from lidiff_b200.engine import Geometry
    h = H()
    pts, coords = random_field(40_000, spread, 17)
    N = coords.shape[0]
    g = Geometry(h, N)
    g.build(coords.to(DEV).contiguous(), N)
    sizes = g.sizes()
    gen = torch.Generator().manual_seed(1)
    for (nbr, perm, lvl, kvol) in ((g.nbr3[0], g.perm3[0], 0, 27), (g.nbr3[2], g.perm3[2], 2, 27), (g.nbr_dn[1], g.perm_dn[1], 1, 8),
                                   (g.nbr_up[0], g.perm_up[0], 0, 8)):
        M = sizes[lvl]
        p = perm[:M].cpu().numpy()
        assert np.array_equal(np.sort(p), np.arange(M)), "not a permutation"
        mask = ((nbr[:, :M] >= 0).long() << torch.arange(kvol, device=DEV)[:, None]).sum(0).cpu().numpy()
        if kvol == 8:
            assert (np.diff(mask[p]) >= 0).all(), "8-bit masks must come out sorted"
        else:
            centre_only = mask[p] == (1 << 13)
            assert centre_only[: centre_only.sum()].all(), "centre-only rows first"
            ms = mask[p].astype(np.int64)
            extras = ms & ~(1 << 13)
            key = ((np.array([bin(int(v)).count("1") for v in extras]) >= 2).astype(np.int64) << 26) | ((ms >> 14) << 13) | (ms & 0x1FFF)
            assert (np.diff(key) >= 0).all(), "27-bit masks must come out sorted by [>=2 neighbours | mask]"
            if lvl in g.morton_levels:          # rows of equal mask in Morton order of (x,y,z) >> level (9 bits per axis)
                C = g.C[lvl][:M].cpu().numpy().astype(np.int64)[p]

                def part(v):
                    v = v & 0x1FF
                    out = np.zeros_like(v)
                    for b in range(9):
                        out |= ((v >> b) & 1) << (3 * b)
                    return out
                code = part(C[:, 1] >> lvl) | (part(C[:, 2] >> lvl) << 1) | (part(C[:, 3] >> lvl) << 2)
                same = np.diff(key) == 0
                assert (np.diff(code)[same] >= 0).all(), "rows of equal mask must be in Morton order"
        cin, cout = 32, 64
        W = (torch.randn(kvol, cin, cout, generator=gen) * 0.1).to(DEV)
        x = torch.randn(N, cin, generator=gen).to(DEV)
        outs = []
        for use_perm in (False, True):
            out = torch.zeros(N, cout, device=DEV)
            d = ConvDesc()
            d.c1, d.c2, d.cout, d.kvol = cin, 0, cout, kvol
            d.weight = W.data_ptr()
            wp = h.pack_weights(W) if algo == 2 else None
            d.weight_packed = wp.data_ptr() if wp is not None else None
            d.nbr, d.nbr_stride, d.d_mout, d.mout_cap, d.npass = nbr.data_ptr(), N, g.d_n[lvl].data_ptr(), N, 1
            d.row_perm = perm.data_ptr() if use_perm else None
            d.io[0] = ConvIO(x.data_ptr(), None, None, out.data_ptr(), None, None, None)
            h.spconv(d, algo)
            outs.append(out[:M].clone())
        if algo == 1:
            assert torch.equal(outs[0], outs[1]), "row order changed the result"
        else:   # the tensor-core variant groups a tile's offsets for its two-level accumulation: same sum, other rounding
            assert rel_err(outs[1], outs[0]) < 1e-5, "row order changed the result"


def test_nn_match_grid_equals_brute_force():
    """shell search over the key lattice == exhaustive argmin incl. lowest-index ties and far-away fallback"""
    from lidiff_b200.engine import Geometry
    h = H()
    g = torch.Generator().manual_seed(4)
    # keys: occupied stride-16 cells of a noisy "scan"; queries: near, on ties, and far outside
    base = torch.randn(7_000, 3, generator=g) * torch.tensor([400.0, 400.0, 40.0])        # <= 8192 key cells: table path
    kc = torch.cat([torch.zeros(base.shape[0], 1), torch.round(base)], 1)
    geo = Geometry(h, kc.shape[0], with_up=False)
    geo.build(kc.to(DEV).contiguous(), kc.shape[0])
    nk = geo.sizes()[4]
    keys = geo.C[4][:nk]
    q_near = torch.round(base[:7_000].repeat(3, 1) + torch.randn(21_000, 3, generator=g) * 20)
    q_tie = keys[:2_000, 1:].cpu().float() + 8.0                         # exactly between lattice cells
    q_far = torch.round(torch.randn(3_000, 3, generator=g) * 3000)
    q = torch.cat([q_near, q_tie, q_far], 0)
    q = torch.cat([torch.zeros(q.shape[0], 1), q], 1).int().to(DEV).contiguous()
    a = torch.empty(q.shape[0], dtype=torch.int32, device=DEV)
    b = torch.empty_like(a)
    h.nn_match(q, None, q.shape[0], keys, geo.d_n[4], kc.shape[0], 0, a)
    h.nn_match_grid(q, None, q.shape[0], geo.C[4], geo.d_n[4], kc.shape[0], geo.grid[4], 16, 4, b)
    assert torch.equal(a, b)
    c = torch.empty_like(a)
    tab = h.nn_table(geo.C[4], geo.d_n[4], kc.shape[0])
    h.nn_match_table(q, None, q.shape[0], geo.C[4], geo.d_n[4], kc.shape[0], tab, 16, 4, c)
    assert torch.equal(a, c), "shared-memory table variant"
    t = torch.empty_like(a)
    tree = h.nn_tree(geo.C[4], geo.d_n[4], kc.shape[0])
    h.nn_match_tree(q, None, q.shape[0], tree, kc.shape[0], t)
    assert torch.equal(a, t), "bounding-box hierarchy variant"
    ref = ome.match_part_to_full(q[:5000].cpu(), keys.cpu())
    assert torch.equal(a[:5000].long().cpu(), ref)


def test_nn_match_tree_batches_ties_and_degenerate_sets():
    """lb2_nn_match_tree == exhaustive argmin for multi-batch keys, duplicated coordinates (lowest row wins), a single key"""
    h = H()
    g = torch.Generator().manual_seed(9)
    for nk, nb in ((1, 1), (5, 1), (3000, 3), (4097, 2)):
        kxyz = torch.randint(-60, 60, (nk, 3), generator=g) * 16
        kxyz[nk // 2:] = kxyz[: nk - nk // 2].clone()                 # duplicated coordinates
        kb = torch.randint(0, nb, (nk, 1), generator=g)
        keys = torch.cat([kb, kxyz], 1).int().to(DEV).contiguous()
        q = torch.cat([torch.randint(0, nb + 1, (20_000, 1), generator=g), torch.randint(-1500, 1500, (20_000, 3), generator=g)], 1).int().to(DEV).contiguous()
        a = torch.empty(q.shape[0], dtype=torch.int32, device=DEV)
        t = torch.empty_like(a)
        d_nk = torch.tensor([nk], dtype=torch.int32, device=DEV)
        cap = nk + 100                                                 # capacity above the live count
        kpad = torch.cat([keys, torch.full((100, 4), 7, dtype=torch.int32, device=DEV)], 0).contiguous()
        h.nn_match(q, None, q.shape[0], kpad, d_nk, cap, 0, a)
        tree = h.nn_tree(kpad, d_nk, cap)
        h.nn_match_tree(q, None, q.shape[0], tree, cap, t)
        assert torch.equal(a, t), (nk, nb)
        hint = torch.randint(0, nk, (777,), generator=g).int().to(DEV)            # arbitrary (even bad) hints never change the answer
        hof = torch.randint(0, 777, (q.shape[0],), generator=g).int().to(DEV)
        t2 = torch.empty_like(a)
        h.nn_match_tree(q, None, q.shape[0], tree, cap, t2, kpad, hof, hint)
        assert torch.equal(a, t2), ("hinted", nk, nb)


@pytest.mark.parametrize("c1,c2,cout,lvl,spread", [(32, 0, 32, 0, 1.0), (96, 32, 96, 1, 0.3), (128, 64, 128, 2, 0.3), (64, 0, 64, 2, 1.0), (128, 0, 128, 0, 0.05)])
def test_scatter_split_equals_output_stationary_conv(c1, c2, cout, lvl, spread, monkeypatch):
    """gather-GEMM-scatter (off-centre pairs) + centre 1x1 conv with pre_add == the plain 3^3 convolution, two passes"""
    monkeypatch.setenv("LB2_SCATTER_LEVELS", "012")            # pair lists for every sparse level in this test
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO, ScatterDesc
    from lidiff_b200.engine import Geometry
    h = H()
    pts, coords = random_field(60_000, spread, 23)
    N = coords.shape[0]
    g = Geometry(h, N)
    g.build(coords.to(DEV).contiguous(), N)
    M = g.sizes()[lvl]
    koff = g.koff[lvl].cpu().numpy()
    nbr = g.nbr3[lvl][:, :M].cpu().numpy()
    # pair lists: same pair sets as the neighbour table, centre skipped
    pin, pout = g.pair_in[lvl].cpu().numpy(), g.pair_out[lvl].cpu().numpy()
    for k in range(27):
        got = set(zip(pin[koff[k]:koff[k + 1]].tolist(), pout[koff[k]:koff[k + 1]].tolist()))
        o = np.nonzero(nbr[k] >= 0)[0]
        ref = set() if k == 13 else set(zip(nbr[k][o].tolist(), o.tolist()))
        assert got == ref, k
    gen = torch.Generator().manual_seed(c1 + cout)
    ctot = c1 + c2
    W = (torch.randn(27, ctot, cout, generator=gen) / np.sqrt(ctot * 27)).to(DEV)
    A = torch.randn(2, N, c1, generator=gen).to(DEV)
    B = torch.randn(2, N, c2, generator=gen).to(DEV) if c2 else None
    sc_, sh_ = (torch.rand(cout, generator=gen) + 0.5).to(DEV), torch.randn(cout, generator=gen).to(DEV)
    Wp, Wc = h.pack_weights(W), W[13:14].contiguous()
    Wpc = h.pack_weights(Wc)

    def conv(kvol, weight, packed, nbr_t, pre, out):
        d = ConvDesc()
        d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, kvol
        d.weight, d.weight_packed = weight.data_ptr(), packed.data_ptr()
        d.scale, d.shift, d.relu = sc_.data_ptr(), sh_.data_ptr(), 1
        d.nbr = nbr_t.data_ptr() if nbr_t is not None else None
        d.nbr_stride, d.d_mout, d.mout_cap, d.npass = N, g.d_n[lvl].data_ptr(), N, 2
        for p in range(2):
            d.io[p] = ConvIO(A[p].data_ptr(), B[p].data_ptr() if B is not None else None, None, out[p].data_ptr(), None, None, None,
                             pre[p].data_ptr() if pre is not None else None)
        h.spconv(d, _lib.ALGO_TC)

    ref = torch.zeros(2, N, cout, device=DEV)
    conv(27, W, Wp, g.nbr3[lvl], None, ref)
    pre = torch.full((2, N, cout), 7.0, device=DEV)               # must be cleared by the kernel
    sd = ScatterDesc()
    sd.c1, sd.c2, sd.cout, sd.kvol, sd.npass = c1, c2, cout, 27, 2
    sd.weight_packed = Wp.data_ptr()
    sd.pair_in, sd.pair_out = g.pair_in[lvl].data_ptr(), g.pair_out[lvl].data_ptr()
    sd.koff, sd.tile_off = g.koff[lvl].data_ptr(), g.tile_off[lvl].data_ptr()
    for p in range(2):
        sd.in1[p], sd.in2[p], sd.out[p] = A[p].data_ptr(), (B[p].data_ptr() if B is not None else None), pre[p].data_ptr()
    sd.d_zero_rows, sd.zero_rows_cap = g.d_n[lvl].data_ptr(), N
    assert h.scatter_supported(c1, c2, cout, 27)
    h.spconv_scatter(sd)
    out = torch.zeros(2, N, cout, device=DEV)
    conv(1, Wc, Wpc, None, pre, out)
    e = rel_err(out[:, :M], ref[:, :M])
    print(f"scatter split {c1}+{c2}->{cout} L{lvl}: pairs {koff[27]}, rel err vs output-stationary {e:.2e}")
    assert e < 2e-5


@pytest.mark.parametrize("c1,c2,cout", [(64, 0, 64), (96, 32, 96), (256, 128, 256)])
def test_split_companion_inputs_give_identical_results(c1, c2, cout):
    """fp16 hi/lo companions + cp.async gather == fp32 inputs split in registers (same rounding), and the epilogue's
    out_h is the split of its fp32 output"""
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    from lidiff_b200.engine import Geometry
    h = H()
    pts, coords = random_field(30_000, 0.4, 29)
    N = coords.shape[0]
    g = Geometry(h, N)
    g.build(coords.to(DEV).contiguous(), N)
    M = g.sizes()[0]
    gen = torch.Generator().manual_seed(3)
    W = (torch.randn(27, c1 + c2, cout, generator=gen) * 0.05).to(DEV)
    Wp = h.pack_weights(W)
    ones = torch.ones(1, max(c1, c2, 1), device=DEV)
    xs, xh = [], []
    for c in (c1, c2):
        if c == 0:
            xs.append(None); xh.append(None); continue
        x = (torch.randn(N, c, generator=gen) * 3).to(DEV)
        y, yh = torch.empty_like(x), torch.zeros(N, 2 * c, dtype=torch.float16, device=DEV)
        h.gate_mul(x, ones[:, :c].contiguous(), None, None, N, c, y, yh)            # y = x * 1, yh = split(y)
        assert torch.equal(y, x)
        hi, lo = yh[:, :c].float(), yh[:, c:].float()
        assert torch.equal(hi, x.half().float()) and (hi + lo - x).abs().max() <= 2e-6 * x.abs().max()
        xs.append(x); xh.append(yh)
    outs = []
    for use_h in (False, True):
        out = torch.zeros(N, cout, device=DEV)
        out_h = torch.zeros(N, 2 * cout, dtype=torch.float16, device=DEV)
        d = ConvDesc()
        d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, 27
        d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
        d.nbr, d.nbr_stride, d.d_mout, d.mout_cap, d.npass = g.nbr3[0].data_ptr(), N, g.d_n[0].data_ptr(), N, 1
        d.io[0] = ConvIO(xs[0].data_ptr(), xs[1].data_ptr() if xs[1] is not None else None, None, out.data_ptr(), None, None, None, None,
                         xh[0].data_ptr() if use_h else None, (xh[1].data_ptr() if (use_h and xh[1] is not None) else None),
                         out_h.data_ptr(), None)
        h.spconv(d, _lib.ALGO_TC)
        outs.append((out[:M].clone(), out_h[:M].clone()))
    assert torch.equal(outs[0][0], outs[1][0]), "cp.async split path differs from the register path"
    o, oh = outs[1]
    assert torch.equal(oh[:, :cout].float(), o.half().float())
    assert (oh[:, :cout].float() + oh[:, cout:].float() - o).abs().max() <= 2e-6 * o.abs().max()


@pytest.mark.parametrize("c1,c2,cout,lvl,kind", [(32, 0, 32, 0, "3"), (96, 32, 96, 1, "3"), (128, 0, 128, 2, "3"), (256, 128, 256, 3, "3"),
                                                    (256, 0, 256, 3, "up"), (128, 0, 128, 4, "dn"), (384, 0, 256, 3, "1"),
                                                    (64, 0, 64, 2, "3"), (128, 64, 128, 2, "3"), (64, 0, 128, 3, "3"), (32, 0, 64, 2, "1")])
def test_persistent_kernel_equals_per_tile_kernel(c1, c2, cout, lvl, kind):
    """LB2_ALGO_TC and LB2_ALGO_TC_TILE run the same math in the same order: identical results, with row order, two passes,
    fused epilogue and split outputs"""
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    from lidiff_b200.engine import Geometry
    h = H()
    pts, coords = random_field(70_000, 1.0 if lvl >= 3 else 0.3, 31)
    N = coords.shape[0]
    g = Geometry(h, N)
    g.build(coords.to(DEV).contiguous(), N)
    M = g.sizes()[lvl]
    nbr, perm, kvol = {"3": (g.nbr3[lvl], g.perm3[lvl], 27), "up": (g.nbr_up[lvl], g.perm_up[lvl], 8),
                       "dn": (g.nbr_dn[lvl], g.perm_dn[lvl], 8), "1": (None, None, 1)}[kind]
    gen = torch.Generator().manual_seed(c1 + cout + lvl)
    W = (torch.randn(kvol, c1 + c2, cout, generator=gen) / np.sqrt((c1 + c2) * kvol)).to(DEV)
    Wp = h.pack_weights(W)
    A = torch.randn(2, N, c1, generator=gen).to(DEV)
    B = torch.randn(2, N, c2, generator=gen).to(DEV) if c2 else None
    R = torch.randn(2, N, cout, generator=gen).to(DEV)
    sc_, sh_ = (torch.rand(cout, generator=gen) + 0.5).to(DEV), torch.randn(cout, generator=gen).to(DEV)
    tab = torch.randn(40, cout, generator=gen).to(DEV)
    gi = torch.randint(0, 40, (N,), generator=gen, dtype=torch.int32).to(DEV)

    def split_of(x):                                   # fp16 hi/lo companion through the library's own split (gate_mul by 1)
        if x is None:
            return None
        c = x.shape[-1]
        one = torch.ones(1, c, device=DEV)
        xh = torch.zeros(2, N, 2 * c, dtype=torch.float16, device=DEV)
        for p_ in range(2):
            h.gate_mul(x[p_], one, None, None, N, c, torch.empty_like(x[p_]), xh[p_])
        return xh
    A_h, B_h = split_of(A), split_of(B)                # with companions the 256-channel layers take the register-total kernel
    res = []
    for algo in (_lib.ALGO_TC_TILE, _lib.ALGO_TC):
        out, outg = torch.zeros(2, N, cout, device=DEV), torch.zeros(2, N, cout, device=DEV)
        out_h = torch.zeros(2, N, 2 * cout, dtype=torch.float16, device=DEV)
        d = ConvDesc()
        d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, kvol
        d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
        d.scale, d.shift, d.relu = sc_.data_ptr(), sh_.data_ptr(), 1
        d.nbr = nbr.data_ptr() if nbr is not None else None
        d.nbr_stride, d.d_mout, d.mout_cap, d.npass = N, g.d_n[lvl].data_ptr(), N, 2
        d.row_perm = perm.data_ptr() if perm is not None else None
        d.row_mask = g.mask_of[nbr.data_ptr()].data_ptr() if nbr is not None else None     # persistent kernels skip absent offsets' index loads
        for p_ in range(2):
            d.io[p_] = ConvIO(A[p_].data_ptr(), B[p_].data_ptr() if B is not None else None, R[p_].data_ptr(), out[p_].data_ptr(),
                              tab.data_ptr(), gi.data_ptr() if p_ == 0 else None, outg[p_].data_ptr(), None,
                              A_h[p_].data_ptr(), B_h[p_].data_ptr() if B_h is not None else None, out_h[p_].data_ptr(), None)
        h.spconv(d, algo)
        res.append((out[:, :M].clone(), outg[:, :M].clone(), out_h[:, :M].clone()))
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)
    assert res[0][0].abs().sum() > 0
