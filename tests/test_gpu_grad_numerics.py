"""The training gradients at their edges, element by element against fp64, under the error model of tests/grad_numerics.py:
  * lb2_spconv_wgrad over row counts at the stage, group and chunk edges (and one bench-sized layer), every channel shape class,
    designed stage patterns, operand magnitudes, non-finite values, determinism and rejected shapes;
  * the input gradient of every adjoint kind through the ME surface, against fp64 autograd of a gather-GEMM;
  * rowsum.index_sum and lb2_segment_sum bit for bit against a sequential host sum, and the backwards built on them;
  * reset_parameters() after a forward refreshes the packed weights.
Each numerics case prints a NUMERICS line (-s) with both normalised errors next to their bars."""
import math

import numpy as np
import pytest
import torch

import grad_numerics as gn
import split_numerics as sn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def handle():
    from lidiff_b200 import _lib
    return _lib.get_handle(DEV)


def wgrad(X, G, nbr, kvol):
    dw = torch.full((kvol, X.shape[1], G.shape[1]), math.nan, device=DEV)
    handle().spconv_wgrad(X, G, nbr, kvol, dw)
    return dw


def check_wgrad(name, X, G, nbr, kvol):
    """one launch against the fp64 reference on the device: both bars, every element; returns (dw, reference)"""
    X, G = X.to(DEV), G.to(DEV)
    nbr = nbr.to(DEV).contiguous() if nbr is not None else None
    dw = wgrad(X, G, nbr, kvol)
    ref = gn.WgradReference(X, G, nbr, kvol)
    eh, es = ref.errors(dw)
    m = G.shape[0]
    print(f"NUMERICS wgrad {name}: hard {eh:.3f} of bound (tau_h {gn.tau_h(m):.2e}), stat {es:.2e} (tau_s {gn.tau_s(m):.2e})")
    assert eh <= 1.0, name
    assert es <= gn.tau_s(m), name
    return dw, ref


# ---- weight gradient: row counts x channel shapes x kernel volumes -------------------------------------------------------------
ROWS = [1, 2, 63, 64, 65, 319, 320, 321, 8191, 8192, 8193, 131071, 131073]
SHAPES = [(1, 32), (3, 64), (5, 96), (8, 128), (16, 256), (40, 32), (96, 64), (128, 96), (192, 128), (384, 256), (512, 64)]
KVOLS = [1, 8, 27]
ROW_CASES = [(m, *SHAPES[(i + j * 6) % len(SHAPES)], KVOLS[(i + j) % 3]) for i, m in enumerate(ROWS) for j in range(2)]


def _rows_operands(m, cin, cout, kvol, seed, p=0, gmax=1e-4, col_scale=False, density=None):
    m_in = m if kvol == 1 else m + 17
    X, G = gn.operands(m_in, m, cin, cout, p, gmax, seed, col_scale)
    nbr = None if kvol == 1 else gn.random_nbr(m, m_in, kvol, density or (0.3 if kvol == 27 else 0.5), seed + 1)
    return X, G, nbr


@pytest.mark.parametrize("m,cin,cout,kvol", ROW_CASES, ids=lambda v: str(v))
def test_wgrad_row_counts_and_shapes(m, cin, cout, kvol):
    X, G, nbr = _rows_operands(m, cin, cout, kvol, m * 3 + cin + cout + kvol)
    check_wgrad(f"m{m}_{cin}to{cout}_k{kvol}", X, G, nbr, kvol)


def test_wgrad_bench_sized_layer():
    """the level-0 row count of scripts/bench_train_refine.py (1 029 259 rows: 16 chunks of 64 384 rows), 27: 96 -> 96"""
    m = 1_029_259
    assert gn.nchunks_of(m) == 16 and gn.rows_per_chunk_of(m) == 64_384
    X, G, nbr = _rows_operands(m, 96, 96, 27, 11, density=0.3)
    check_wgrad(f"m{m}_96to96_k27", X, G, nbr, 27)


# ---- stage patterns ---------------------------------------------------------------------------------------------------------
PATTERN_M = 2 * 8192 + 100          # 3 chunks of 5504 rows (86 stages), the last one ends in a partial stage


def pattern_table(m, m_in, seed):
    """(8, m) table, one stage pattern per offset (stages of 64 rows, counted within each chunk)"""
    rpc = gn.rows_per_chunk_of(m)
    o = torch.arange(m)
    st = (o % rpc) // gn.BR
    g = torch.Generator().manual_seed(seed)
    rnd = torch.randint(0, m_in, (8, m), generator=g, dtype=torch.int32)
    none = torch.full((m,), -1, dtype=torch.int32)
    nbr = torch.stack([
        none,                                                        # 0: every stage empty
        torch.where(st % 2 == 0, rnd[1], none),                      # 1: live and empty stages alternate
        torch.where(st % 3 == 0, rnd[2], none),                      # 2: a group of 5 live stages spans 10 empty ones
        torch.where(st < 7, rnd[3], none),                           # 3: a group and 2 live stages, then empty to the chunk's end
        torch.where((o == m - 1) | (o == rpc - 1), rnd[4], none),    # 4: one live row in the last (partial) stage of a chunk
        torch.where(o % 2 == 0, torch.full_like(rnd[5], 7), none),   # 5: one input row read by half the output rows
        torch.where(torch.rand(m, generator=g) < 0.5, rnd[6], none),
        torch.where(torch.rand(m, generator=g) < 0.04, rnd[7], none),   # sparse: some stages empty by chance
    ])
    return nbr


@pytest.mark.parametrize("cin,cout", [(64, 64), (40, 96), (256, 32)])
def test_wgrad_stage_patterns(cin, cout):
    m = PATTERN_M
    assert gn.nchunks_of(m) == 3 and m % gn.rows_per_chunk_of(m) % gn.BR != 0
    X, G = gn.operands(m, m, cin, cout, 0, 1e-4, cin + cout)
    nbr = pattern_table(m, m, cin)
    dw, _ = check_wgrad(f"patterns_{cin}to{cout}", X, G, nbr, 8)
    assert (dw[0].view(torch.int32) == 0).all(), "an offset with no neighbour must give +0"


# ---- magnitudes -------------------------------------------------------------------------------------------------------------
MAG_M = 3000


@pytest.mark.parametrize("p", [-24, -12, -4, 0, 8, 15, "edge"])
def test_wgrad_activation_magnitudes(p):
    X, G, nbr = _rows_operands(MAG_M, 64, 64, 8, 101, p=0 if p == "edge" else p)
    if p == "edge":
        e = sn.edge_values()
        e = e[torch.isfinite(e) & (e.abs() < gn.SPLIT_INF)]
        X = e[torch.randint(0, e.numel(), X.shape, generator=torch.Generator().manual_seed(5))]
    check_wgrad(f"x2^{p}", X, G, nbr, 8)


GMAX = [1e-30, 2.0 ** -120, 1e-8, 1e-4, 1.0, 1e6, 1e30]


@pytest.mark.parametrize("col_scale", [False, True])
@pytest.mark.parametrize("gmax", GMAX, ids=lambda v: f"{v:g}")
def test_wgrad_gradient_magnitudes(gmax, col_scale):
    """max|G| from 1e-30 to 1e30 (2^-120: the pre-scale stops at 2^126); with col_scale output column n is 2^e_n times the others,
    e_n in -10 .. 10, the pre-scale follows the largest column and every element stays inside its own bound"""
    X, G, nbr = _rows_operands(MAG_M, 64, 96, 8, 202, gmax=gmax, col_scale=col_scale)
    check_wgrad(f"gmax{gmax:g}{'_col' if col_scale else ''}", X, G, nbr, 8)


# ---- non-finite values ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("what", ["x", "g_inf", "g_nan"])
def test_wgrad_non_finite_values_reach_exactly_their_elements(what):
    """NaN / +-inf (and the split's non-finite |x| >= 131024) in X rows, or single +-inf / NaN elements of G: the non-finite dW
    elements are the fp64 reference's, and every other element has the bits of a run with those entries zeroed"""
    X, G, nbr = _rows_operands(MAG_M, 64, 64, 8, 303)
    X0, G0 = X.clone(), G.clone()
    Xb, Gb = X.clone(), G.clone()
    if what == "x":
        X0[[11, 500, 901]] = 0
        Xb[[11, 500, 901]] = 0
        Xb[11, :32] = math.nan
        Xb[500, ::2] = math.inf
        Xb[500, 1::4] = -math.inf
        Xb[901, 5], Xb[901, 6], Xb[901, 7] = 1e30, 2.0 ** 17, -131008.0        # the last one is finite under the split
        X0[901, 7] = -131008.0
    else:
        v = math.nan if what == "g_nan" else math.inf
        for o, j, s in ((40, 3, 1.0), (2000, 10, -1.0), (2999, 63, 1.0)):
            G0[o, j] = 0
            Gb[o, j] = v * s
    nb = nbr.to(DEV)
    dw = wgrad(Xb.to(DEV), Gb.to(DEV), nb, 8)
    dw0 = wgrad(X0.to(DEV), G0.to(DEV), nb, 8)
    ref = gn.WgradReference(Xb.to(DEV), Gb.to(DEV), nb, 8)
    bad = ~torch.isfinite(ref.y)
    print(f"NUMERICS wgrad non-finite {what}: {int(bad.sum())} of {bad.numel()} elements non-finite in the reference")
    assert bad.any() and (~bad).any()
    assert torch.equal(~torch.isfinite(dw), bad), "non-finite elements differ from the fp64 reference's"
    assert sn.same_bits(dw[~bad], dw0[~bad]), "an element that reads no non-finite value changed"


# ---- determinism and independence -------------------------------------------------------------------------------------------
def test_wgrad_bits_do_not_depend_on_reruns_stride_or_unread_rows():
    m, m_in, kvol = 8193 + 64, 9000, 8
    X, G = gn.operands(m_in, m, 64, 64, 0, 1e-4, 404)
    nbr = gn.random_nbr(m, m, kvol, 0.5, 405)                           # reads only rows < m
    X, G, nb = X.to(DEV), G.to(DEV), nbr.to(DEV)
    a = wgrad(X, G, nb, kvol)
    assert sn.same_bits(a, wgrad(X, G, nb, kvol))
    buf = torch.randint(0, m, (kvol, m + 333), dtype=torch.int32, device=DEV)      # valid-looking entries past m_out
    buf[:, :m] = nb
    assert sn.same_bits(a, wgrad(X, G, buf[:, :m], kvol))
    unread = torch.ones(m_in, dtype=torch.bool, device=DEV)
    unread[nb[nb >= 0].long()] = False
    assert unread.sum() > m_in - m
    Xu = X.clone()
    Xu[unread] = math.nan
    assert sn.same_bits(a, wgrad(Xu, G, nb, kvol))


def test_wgrad_no_rows_gives_zeros():
    for kvol, nbr in ((1, None), (8, torch.empty(8, 0, dtype=torch.int32, device=DEV))):
        dw = wgrad(torch.randn(10, 64, device=DEV), torch.empty(0, 32, device=DEV), nbr, kvol)
        assert (dw.view(torch.int32) == 0).all()


@pytest.mark.parametrize("kvol,cin,cout", [(1, 0, 32), (1, 9, 32), (1, 513, 32), (1, 64, 48), (1, 64, 160), (1, 64, 512),
                                           (2, 64, 64)])
def test_wgrad_rejects_unsupported_shapes_before_any_launch(kvol, cin, cout):
    h = handle()
    m = 64
    X, G = torch.zeros(m, cin, device=DEV), torch.zeros(m, cout, device=DEV)
    nbr = None if kvol == 1 else torch.zeros(kvol, m, dtype=torch.int32, device=DEV)
    dw = torch.full((kvol, cin, cout), 5.0, device=DEV)
    torch.cuda.synchronize()
    n0 = h.launch_count()
    with pytest.raises(RuntimeError):
        h.spconv_wgrad(X, G, nbr, kvol, dw)
    torch.cuda.synchronize()
    assert h.launch_count() == n0
    assert (dw == 5.0).all()


# ---- input gradients through the ME surface ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cm():
    from lidiff_b200 import me as ME
    g = torch.Generator().manual_seed(2024)
    pts = torch.randn(40_000, 3, generator=g) * torch.tensor([0.5, 0.5, 0.12])
    coords = torch.cat([torch.zeros(pts.shape[0], 1), torch.round(pts / 0.05)], 1)
    field = ME.TensorField(pts.to(DEV), coords.to(DEV))
    field.sparse()
    return field.coordinate_manager


# name: (class, cin, cout, kernel_size, stride, tensor stride of the input)
KINDS = {"3x3x3": ("conv", 64, 64, 3, 1, 1), "k2s2": ("conv", 32, 64, 2, 2, 1), "transposed": ("transpose", 256, 128, 2, 2, 2),
         "1x1_matrix": ("conv", 128, 256, 1, 1, 1), "1x1_volume": ("volume1", 128, 96, 1, 1, 1),
         "384to256": ("conv", 384, 256, 3, 1, 2), "192to128": ("conv", 192, 128, 3, 1, 2)}


def make_layer(kind, seed=0):
    from lidiff_b200 import me as ME
    cls, cin, cout, ks, stride, ts = KINDS[kind]
    torch.manual_seed(seed)
    Cls = ME.MinkowskiConvolutionTranspose if cls == "transpose" else ME.MinkowskiConvolution
    layer = Cls(cin, cout, kernel_size=ks, stride=stride, dimension=3).to(DEV)
    if cls == "volume1":                # the (1, cin, cout) form of a 1x1 kernel
        layer.kernel = torch.nn.Parameter(layer.kernel.detach()[None].clone())
    return layer


def forward_map(cm, kind):
    cls, cin, cout, ks, stride, ts = KINDS[kind]
    if ks == 1:
        return None, cm.level(ts).n
    if cls == "transpose":
        return cm.kernel_map(ts, ks, stride, True), cm.level(ts // stride).n
    return cm.kernel_map(ts, ks, stride, False), cm.level(ts * stride).n


def run_layer(layer, cm, ts, X, G):
    """(y, dX, dW) of one forward and backward with output gradient G"""
    from lidiff_b200 import me as ME
    layer.kernel.grad = None
    Xp = X.clone().requires_grad_(True)
    y = layer(ME.SparseTensor(Xp, coordinate_manager=cm, tensor_stride=ts))
    y.F.backward(G)
    return y.F.detach(), Xp.grad.detach(), layer.kernel.grad.detach().clone()


def dgrad_case(cm, kind, gmax, col_scale=False, seed=0):
    cls, cin, cout, ks, stride, ts = KINDS[kind]
    nbr, m_out = forward_map(cm, kind)
    m_in = cm.level(ts).n
    X, G = gn.operands(m_in, m_out, cin, cout, 0, gmax, seed, col_scale)
    return nbr, m_in, X.to(DEV), G.to(DEV)


def check_dgrad(cm, kind, gmax, col_scale=False):
    cls, cin, cout, ks, stride, ts = KINDS[kind]
    layer = make_layer(kind)
    nbr, m_in, X, G = dgrad_case(cm, kind, gmax, col_scale, seed=cin + cout)
    _, dx, _ = run_layer(layer, cm, ts, X, G)
    W = layer.kernel.detach()
    W = W[None] if W.dim() == 2 else W
    cuts = {384: (0, 256, 384), 192: (0, 128, 192)}.get(cin, (0, cin))
    ref = gn.DgradReference(G, W, nbr, m_in, cuts)
    eh, es = ref.errors(dx)
    th, ts_ = ref.bounds()
    print(f"NUMERICS dgrad {kind} gmax{gmax:g}{'_col' if col_scale else ''}: hard {eh:.3f} of bound (tau_h {th:.2e}), "
          f"stat {es:.2e} (tau_s {ts_:.2e})")
    assert eh <= 1.0 and es <= ts_


@pytest.mark.parametrize("col_scale", [False, True])
@pytest.mark.parametrize("kind", list(KINDS))
def test_input_gradient_every_adjoint_kind(cm, kind, col_scale):
    check_dgrad(cm, kind, 1e-3, col_scale)


@pytest.mark.parametrize("gmax", [1e-40] + GMAX, ids=lambda v: f"{v:g}")
@pytest.mark.parametrize("kind", ["3x3x3", "transposed", "384to256"])
def test_input_gradient_magnitudes(cm, kind, gmax):
    """max|G| from a subnormal 1e-40 to 1e30: the power-of-two scale (capped at 2^126) keeps every element inside its bound"""
    check_dgrad(cm, kind, gmax)


@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("kind", ["3x3x3", "1x1_matrix", "transposed"])
def test_input_gradient_non_finite_rows(cm, kind, bad):
    """a NaN or +-inf row of G: the non-finite rows of dX are the fp64 reference's, and every other row has the bits of a run with
    that row zeroed (the scale of G ignores non-finite elements)"""
    cls, cin, cout, ks, stride, ts = KINDS[kind]
    nbr, m_in, X, G = dgrad_case(cm, kind, 1e-3, seed=7)
    r = G.shape[0] // 3
    G0, Gb = G.clone(), G.clone()
    G0[r] = 0
    if bad == "nan":
        Gb[r] = math.nan
    else:
        Gb[r] = torch.where(torch.arange(cout, device=DEV) % 2 == 0, math.inf, -math.inf)
    layer = make_layer(kind)
    _, dx, _ = run_layer(layer, cm, ts, X, Gb)
    _, dx0, _ = run_layer(layer, cm, ts, X, G0)
    W = layer.kernel.detach().double()
    y64 = gn.autograd_dx(Gb.double(), W[None] if W.dim() == 2 else W, nbr, m_in)
    bad_ref = ~torch.isfinite(y64)
    assert bad_ref.any() and (~bad_ref).any()
    assert torch.equal(~torch.isfinite(dx), bad_ref), "non-finite dX elements differ from the fp64 reference's"
    assert sn.same_bits(dx[~bad_ref], dx0[~bad_ref]), "a row that reads no non-finite gradient changed"


def test_reset_parameters_after_a_forward_refreshes_the_packed_weights(cm):
    """forward and backward (the packed forward and adjoint weights are cached), reset_parameters(), then forward, input and
    weight gradient: the same bits as a fresh layer with the new weights"""
    from lidiff_b200 import me as ME
    ts = 1
    nbr, m_in, X, G = dgrad_case(cm, "3x3x3", 1e-3, seed=9)
    layer = make_layer("3x3x3", seed=1)
    run_layer(layer, cm, ts, X, G)
    layer.reset_parameters()
    fresh = ME.MinkowskiConvolution(64, 64, kernel_size=3, stride=1, dimension=3).to(DEV)
    with torch.no_grad():
        fresh.kernel.copy_(layer.kernel)
    for a, b, what in zip(run_layer(layer, cm, ts, X, G), run_layer(fresh, cm, ts, X, G), ("forward", "input gradient", "weight gradient")):
        assert sn.same_bits(a, b), what


# ---- row sums bit for bit ------------------------------------------------------------------------------------------------
LENGTHS = [0, 1, 2, 33, 100_000, 0, 1, 2, 33, 5]


def row_values(n, c, dtype, seed):
    """values that cancel (so the order of the adds shows in the bits) with -0.0, subnormals, +-inf and NaN in some rows"""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, c)) * 10.0 ** rng.integers(-3, 4, (n, 1))
    big = rng.random(n) < 0.3
    v[big] += np.where(rng.random((int(big.sum()), 1)) < 0.5, -1e7, 1e7)
    v = v.astype(dtype)
    tiny = np.finfo(dtype).smallest_subnormal
    specials = {0: -0.0, 1: tiny, 2: -3 * tiny, 3: np.inf, 4: -np.inf, 5: np.nan, 6: np.finfo(dtype).tiny / 2}
    for j, (r, val) in enumerate(zip(rng.integers(0, max(n, 1), len(specials)), specials.values())):
        if n > 40:
            v[r, j % c] = val
    if n > 40:
        v[1:3] = -0.0                  # the segment of length 2 that starts at row 1 holds only -0.0
    return v


def offsets_of(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


@pytest.mark.parametrize("use_order", [False, True])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("c", [1, 3, 31, 32, 33, 96, 100])
def test_segment_sum_is_sequential_bit_for_bit(c, dtype, use_order):
    off = offsets_of(LENGTHS)
    n = int(off[-1])
    v = row_values(n, c, dtype, c * 10 + use_order)
    order = np.random.default_rng(c).permutation(n).astype(np.int64) if use_order else None
    want = gn.sequential_segment_sum(v, order, off)
    out = torch.full((len(LENGTHS), c), math.nan, dtype=torch.from_numpy(v).dtype, device=DEV)
    handle().segment_sum(torch.from_numpy(v).to(DEV), torch.from_numpy(order).to(DEV) if use_order else None,
                         torch.from_numpy(off).to(DEV), out)
    assert gn.same_bits(out.cpu(), torch.from_numpy(want))
    assert (out[0].view(torch.int32 if dtype == np.float32 else torch.int64) == 0).all()      # an empty segment is +0


def test_segment_sum_of_a_million_rows():
    off = offsets_of([3, 1_000_000, 2])
    v = row_values(int(off[-1]), 3, np.float32, 1)
    want = gn.sequential_segment_sum(v, None, off)
    out = torch.empty(3, 3, device=DEV)
    handle().segment_sum(torch.from_numpy(v).to(DEV), None, torch.from_numpy(off).to(DEV), out)
    assert gn.same_bits(out.cpu(), torch.from_numpy(want))


def index_sum_want(v, idx, n):
    order = np.argsort(idx, kind="stable")
    return gn.sequential_segment_sum(v, order, offsets_of(np.bincount(idx, minlength=n)))


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("c", [1, 33, 100])
def test_index_sum_is_sequential_in_row_order(c, dtype):
    from lidiff_b200.rowsum import index_sum
    rng = np.random.default_rng(c)
    n = 500                                              # outputs 0 .. 499; every third is never used
    used = np.array([j for j in range(n) if j % 3])
    idx = np.concatenate([np.full(L, used[i % len(used)]) for i, L in enumerate([1, 2, 33, 20_000] + [7] * 300)])
    idx = idx[rng.permutation(idx.shape[0])]
    v = row_values(idx.shape[0], c, dtype, c)
    out = index_sum(torch.from_numpy(v).to(DEV), torch.from_numpy(idx).to(DEV), n)
    assert gn.same_bits(out.cpu(), torch.from_numpy(index_sum_want(v, idx, n)))
    assert (out[0].cpu().numpy() == 0).all() and not np.signbit(out[0].cpu().numpy()).any()


def test_index_sum_without_rows():
    from lidiff_b200.rowsum import index_sum
    out = index_sum(torch.empty(0, 3, device=DEV), torch.empty(0, dtype=torch.int64, device=DEV), 4)
    assert out.shape == (4, 3) and (out.view(torch.int32) == 0).all()
    assert index_sum(torch.ones(5, 3, device=DEV), torch.zeros(5, dtype=torch.int64, device=DEV), 0).shape == (0, 3)


def test_gather_slice_and_voxel_mean_backwards_equal_their_closed_forms():
    from lidiff_b200 import me as ME
    from lidiff_b200.rowsum import GatherRows
    rng = np.random.default_rng(3)
    # GatherRows: the backward of src[idx] is index_sum
    src = torch.randn(300, 33, device=DEV, requires_grad=True)
    idx = rng.integers(0, 250, 5000)                       # rows 250 .. 299 are never gathered
    grad = row_values(5000, 33, np.float32, 4)
    GatherRows.apply(src, torch.from_numpy(idx).to(DEV)).backward(torch.from_numpy(grad).to(DEV))
    assert gn.same_bits(src.grad.cpu(), torch.from_numpy(index_sum_want(grad, idx, 300)))
    # slice() and sparse(): points with shared voxels
    pts = torch.from_numpy(rng.uniform(-1, 1, (6000, 3)).astype(np.float32))
    coords = torch.cat([torch.zeros(6000, 1), torch.floor(pts / 0.2)], 1)
    F = torch.randn(6000, 5, device=DEV, requires_grad=True)
    field = ME.TensorField(F, coords.to(DEV))
    s = field.sparse()
    inv = field.inverse_mapping.cpu().numpy()
    nvox = s.F.shape[0]
    gs = row_values(nvox, 5, np.float32, 6)
    s.F.backward(torch.from_numpy(gs).to(DEV))
    count = np.bincount(inv, minlength=nvox).astype(np.float32)
    assert gn.same_bits(F.grad.cpu(), torch.from_numpy((gs / count[:, None])[inv]))
    Fv = torch.randn(nvox, 5, device=DEV, requires_grad=True)
    sl = ME.SparseTensor(Fv, coordinate_manager=field.coordinate_manager).slice(field)
    gp = row_values(6000, 5, np.float32, 7)
    sl.F.backward(torch.from_numpy(gp).to(DEV))
    assert gn.same_bits(Fv.grad.cpu(), torch.from_numpy(index_sum_want(gp, inv, nvox)))
