"""Offset split of the 3^3 tensor-core convolutions: a layer with one kernel offset per accumulation group (c1 + c2 >= 176) runs as
G launches over contiguous offset ranges, each over the rows and tiles of its own range order, carrying the fp32 totals through
memory.  The adds are the same as in one launch over all 27 offsets, in the same order, so the split must give the same bytes.

Checked here: lb2_row_order_range / lb2_tile_order_range against a numpy restatement; every split layer shape at G = 2 and 3
against G = 1 on the benchmark scan's geometry; one full engine step at 180 000 points with the split on and off."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- numpy restatement of the range order --------------------------------------------------------------------------------------
def range_key(mask: np.ndarray, k0: int, k1: int) -> np.ndarray:
    """[sub == 0 | 2 or more off-centre bits of sub | sub without the centre bit, compacted to the range], sub = mask & [k0, k1)"""
    m = mask.astype(np.int64)
    sub = m & (((1 << k1) - 1) & ~((1 << k0) - 1))
    bits = [k for k in range(k0, k1) if k != 13]
    local = np.zeros_like(sub)
    for j, k in enumerate(bits):
        local |= ((sub >> k) & 1) << j
    off = sub & ~(1 << 13)
    multi = sum((off >> k) & 1 for k in range(27)) >= 2
    nb = len(bits)
    return ((sub == 0).astype(np.int64) << (nb + 1)) | (multi.astype(np.int64) << nb) | local


def run_range_order(h, mask_np, k0, k1):
    n = mask_np.shape[0]
    mask = torch.from_numpy(mask_np.astype(np.int64).astype(np.uint32).view(np.int32)).to(DEV)
    d_n = torch.tensor([n], dtype=torch.int32, device=DEV)
    perm = torch.full((n,), -7, dtype=torch.int32, device=DEV)
    live = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    scratch = torch.zeros((h.row_order_scratch_bytes(n) + 3) // 4, dtype=torch.int32, device=DEV)
    h.row_order_range(mask, d_n, n, k0, k1, perm, live, scratch)
    order = torch.full(((n + 127) // 128,), -7, dtype=torch.int32, device=DEV)
    tscratch = torch.zeros((n + 127) // 128, dtype=torch.int32, device=DEV)
    h.tile_order_range(mask, perm, live if k1 < 27 else d_n, n, k0, k1, order, tscratch)
    torch.cuda.synchronize()
    return perm.cpu().numpy(), int(live.item()), order.cpu().numpy()


def random_masks(n, seed, p=0.25, centre=True, forbid=0):
    g = np.random.default_rng(seed)
    bits = g.random((n, 27)) < p
    m = (bits * (1 << np.arange(27))).sum(1).astype(np.int64)
    if centre:
        m |= 1 << 13
    return m & ~forbid


@pytest.mark.parametrize("k0,k1,centre,forbid,live", [
    (0, 14, True, 0, "all"), (14, 27, True, 0, None), (0, 9, True, 0, None), (9, 18, True, 0, "all"), (18, 27, True, 0, None),
    (13, 14, True, 0, "all"), (13, 14, False, 0, None), (0, 27, False, 0, None), (5, 6, True, 0, None),
    (20, 27, True, ((1 << 27) - 1) & ~((1 << 20) - 1), "none"),     # an empty range: no row has a bit in it
])
def test_range_row_order_matches_numpy(k0, k1, centre, forbid, live):
    from lidiff_b200 import _lib
    h = _lib.get_handle(DEV)
    n = 70_001
    mask = random_masks(n, k0 * 31 + k1, centre=centre, forbid=forbid)
    mask[::97] = 0                                               # rows without any neighbour (not a self map's, but legal input)
    if centre and live == "all":
        mask[::97] = 1 << 13
    perm, n_live, order = run_range_order(h, mask, k0, k1)
    key = range_key(mask, k0, k1)
    ref = np.argsort(key, kind="stable")
    assert np.array_equal(perm, ref), "range row order differs from the stable sort of the numpy key"
    ref_live = int(((mask & (((1 << k1) - 1) & ~((1 << k0) - 1))) != 0).sum())
    assert n_live == ref_live
    if live == "all":
        assert n_live == n
    if live == "none":
        assert n_live == 0
    # tile order: the tiles of the dispatched rows, most expensive (popcount of the range-restricted OR) first
    m_rows = n_live if k1 < 27 else n
    nt = (m_rows + 127) // 128
    rmask = ((1 << k1) - 1) & ~((1 << k0) - 1)
    sorted_masks = mask[perm]
    cost = np.array([bin(int(np.bitwise_or.reduce(sorted_masks[t * 128:min((t + 1) * 128, m_rows)])) & rmask).count("1") for t in range(nt)])
    assert sorted(order[:nt].tolist()) == list(range(nt))
    assert (order[nt:] == -1).all()
    c = cost[order[:nt]]
    assert (np.diff(c) <= 0).all(), "tiles not in descending cost order"


# ---- split convolutions on the benchmark scan's geometry -------------------------------------------------------------------------
def bench_coords(sigma, seed):
    z = np.load(os.path.join(GOLD, "step_synth180k.npz"))
    pts = torch.tensor(z["part"]).repeat(10, 1).float()
    g = torch.Generator().manual_seed(seed)
    pts = pts + sigma * torch.randn(pts.shape, generator=g)
    return torch.cat([torch.zeros(pts.shape[0], 1), torch.round(pts / 0.05)], 1)


@pytest.fixture(scope="module")
def bench_geometry():
    from lidiff_b200 import _lib
    from lidiff_b200.engine import Geometry
    h = _lib.get_handle(DEV)
    coords = bench_coords(1.0, 5)
    N = coords.shape[0]
    g = Geometry(h, N)
    g.split_groups = {2: {2, 3}, 3: {2, 3}, 4: {2, 3}}
    g.build(coords.to(DEV).contiguous(), N)
    torch.cuda.synchronize()
    return h, g, N


@pytest.mark.parametrize("c1,c2,cout,lvl,npass", [(256, 0, 256, 4, 2), (256, 0, 256, 4, 1), (256, 128, 256, 3, 2), (256, 0, 256, 3, 1),
                                                   (192, 128, 128, 2, 2), (128, 64, 128, 2, 1), (192, 0, 128, 3, 2)])
def test_split_layer_is_byte_identical_to_one_launch(bench_geometry, c1, c2, cout, lvl, npass):
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    from lidiff_b200.engine import one_offset_per_group
    h, g, N = bench_geometry
    assert one_offset_per_group(c1 + c2)
    M = g.sizes()[lvl]
    nbr = g.nbr3[lvl]
    mask = g.mask_of[nbr.data_ptr()][:M].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    gen = torch.Generator().manual_seed(c1 + c2 + cout + lvl + npass)
    W = (torch.randn(27, c1 + c2, cout, generator=gen) / np.sqrt((c1 + c2) * 27)).to(DEV)
    Wp = h.pack_weights(W)
    A = torch.randn(npass, N, c1, generator=gen)
    A[0, 5] = float("nan")                                        # non-finite inputs: every output that reads them stays non-finite
    A[-1, 7, 3] = float("inf")
    A = A.to(DEV)
    B = torch.randn(npass, N, c2, generator=gen).to(DEV) if c2 else None
    R = torch.randn(npass, N, cout, generator=gen).to(DEV)
    gate = (torch.rand(4, cout, generator=gen) + 0.5).to(DEV)
    gidx = torch.randint(0, 4, (N,), generator=gen, dtype=torch.int32).to(DEV)
    sc_, sh_ = (torch.rand(cout, generator=gen) + 0.5).to(DEV), torch.randn(cout, generator=gen).to(DEV)
    part = torch.full((2, N, 256), float("nan"), device=DEV)       # stale contents must never be read

    def run(G):
        out = torch.full((npass, N, cout), float("nan"), device=DEV)
        og = torch.full((npass, N, cout), float("nan"), device=DEV)
        d = ConvDesc()
        d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, 27
        d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
        d.scale, d.shift, d.relu = sc_.data_ptr(), sh_.data_ptr(), 1
        d.nbr, d.nbr_stride, d.mout_cap, d.npass = nbr.data_ptr(), N, N, npass
        d.row_mask = g.mask_of[nbr.data_ptr()].data_ptr()
        for p_ in range(npass):
            d.io[p_] = ConvIO(A[p_].data_ptr(), B[p_].data_ptr() if B is not None else None, R[p_].data_ptr(), out[p_].data_ptr(),
                              gate.data_ptr(), gidx.data_ptr(), og[p_].data_ptr())
        if G == 1:
            d.d_mout, d.row_perm = g.d_n[lvl].data_ptr(), g.perm3[lvl].data_ptr()
            d.tile_order128 = g.tile_order_of[nbr.data_ptr()][0].data_ptr()
            h.spconv(d, _lib.ALGO_TC)
        else:
            for k0, k1, perm_r, live_r, to_r in g.range_of[(nbr.data_ptr(), G)]:
                d.row_perm, d.tile_order128 = perm_r.data_ptr(), to_r.data_ptr()
                d.d_mout = (g.d_n[lvl] if k1 == 27 else live_r).data_ptr()
                d.k0, d.k1 = k0, k1
                d.partial_in = part.data_ptr() if k0 > 0 else None
                d.partial_out = part.data_ptr() if k1 < 27 else None
                h.spconv(d, _lib.ALGO_TC)
        torch.cuda.synchronize()
        return out[:, :M].cpu(), og[:, :M].cpu()

    ref = run(1)
    assert not torch.isnan(ref[0][:, 8:]).all(), "the reference computed nothing"
    for G in (2, 3):
        ranges = [(a, b) for a, b, *_ in g.range_of[(nbr.data_ptr(), G)]]
        # the cases the carry has to get right: rows with nothing in the last range (their totals come from partial_in alone) and,
        # at G = 3, rows with nothing in [0, 9) (they start the middle range from -0)
        assert ((mask >> ranges[-1][0]) == 0).any()
        assert G == 2 or ((mask & ((1 << ranges[0][1]) - 1)) == 0).any()
        got = run(G)
        for r, x in zip(ref, got):
            assert torch.equal(r.view(torch.int32), x.view(torch.int32)), f"G = {G}: outputs differ from one launch"


def test_split_needs_one_offset_per_group(bench_geometry):
    from lidiff_b200 import _lib
    from lidiff_b200._lib import ConvDesc, ConvIO
    h, g, N = bench_geometry
    lvl, c1, cout = 3, 128, 128                                   # 3 * 8 k-steps per offset: two offsets per group
    nbr = g.nbr3[lvl]
    W = torch.zeros(27, c1, cout, device=DEV)
    Wp = h.pack_weights(W)
    A = torch.zeros(1, N, c1, device=DEV)
    out = torch.zeros(1, N, cout, device=DEV)
    part = torch.zeros(2, N, 256, device=DEV)
    d = ConvDesc()
    d.c1, d.c2, d.cout, d.kvol = c1, 0, cout, 27
    d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
    d.nbr, d.nbr_stride, d.mout_cap, d.npass, d.d_mout = nbr.data_ptr(), N, N, 1, g.d_n[lvl].data_ptr()
    d.row_mask = g.mask_of[nbr.data_ptr()].data_ptr()
    d.io[0] = ConvIO(A[0].data_ptr(), None, None, out[0].data_ptr(), None, None, None)
    d.k0, d.k1, d.partial_out = 0, 14, part.data_ptr()
    with pytest.raises(RuntimeError, match="offset range"):
        h.spconv(d, _lib.ALGO_TC)
    with pytest.raises(RuntimeError, match="offset range"):
        h.spconv(d, _lib.ALGO_FFMA)


# ---- one engine step at 180 000 points ------------------------------------------------------------------------------------------
def test_engine_step_is_byte_identical_with_the_split_on_and_off(monkeypatch):
    import importlib.util
    from lidiff_b200.engine import DenoiseEngine
    spec = importlib.util.spec_from_file_location("make_step_goldens", os.path.join(GOLD, "make_step_goldens.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    z = np.load(os.path.join(GOLD, "step_synth180k.npz"))
    sds = mk.seeded_state_dicts(0)
    off = 0
    for key, size in zip(z["bn_keys"].tolist(), z["bn_sizes"].tolist()):
        net, k = key.split("/", 1)
        sds[net][k] = torch.from_numpy(z["bn_vals"][off:off + size].copy()).reshape(sds[net][k].shape)
        off += size
    scan = torch.tensor(z["part"]).repeat(10, 1)[None]
    start, step = mk.noises(scan.shape, 1234)
    N = scan.shape[1]
    res = {}
    for setting in ("1", "2", "3", "stage4=3,up1=2,up2=3"):
        monkeypatch.setenv("LB2_OFFSET_SPLIT", setting)
        eng = DenoiseEngine(sds["enc"], sds["diff"], device=DEV, n_points=N, denoising_steps=int(z["T"]))
        assert bool(eng.split_of) == (setting != "1")
        st = eng.start(scan, scan + start)
        eps = torch.empty((N, 3), device=DEV)
        eng.step(0, st["xa"], st["xb"], st["ca"], st["cb"], st["x_init"], step[0, 0].to(DEV).contiguous(), st["x0s"], eps_out=eps)
        torch.cuda.synchronize()
        res[setting] = (eps.cpu(), st["xb"].cpu())
        del eng, st
        torch.cuda.empty_cache()
    for setting, (e, x) in res.items():
        assert torch.equal(e.view(torch.int32), res["1"][0].view(torch.int32)), f"eps differs at LB2_OFFSET_SPLIT={setting}"
        assert torch.equal(x.view(torch.int32), res["1"][1].view(torch.int32)), f"x_t differs at LB2_OFFSET_SPLIT={setting}"
