"""The coordinate manager (coords.cu) at its edges, bit for bit against the numpy restatement tests/coords_reference.py: scan
sizes up to the 4M-row limit, live counts below the capacity, 1024 batches, rows at the key-range limits, the status bit, every
map and row order of a 500k-point geometry, the stable radix sort at > 512 blocks, the voxel mean's error bound and order
independence, and the shared-memory NN table past its capacity."""
import numpy as np
import pytest
import torch

import coords_reference as cref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LO, HI = cref.AXIS_MIN, cref.AXIS_MAX


def H():
    from lidiff_b200 import _lib
    return _lib.get_handle(DEV)


def i32(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32)).to(DEV)


def f32(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def unique(h, rows, ts=0, n=None, fp=True, n_cap=None):
    """lb2_unique_build on `rows` (fp32 or int32 input), first n live -> (coords (M, 4), inverse (n_cap,), M, status)"""
    n_cap = rows.shape[0] if n_cap is None else n_cap
    grid = h.new_grid(n_cap)
    out = torch.full((n_cap, 4), 77, dtype=torch.int32, device=DEV)
    inv = torch.full((n_cap,), -7, dtype=torch.int32, device=DEV)
    d_n = torch.zeros(1, dtype=torch.int32, device=DEV)
    d_in = None if n is None else i32([n])
    src = f32(rows) if fp else i32(rows)
    h.unique_build(src if fp else None, None if fp else src, d_in, n_cap, ts, grid, out, inv, d_n, h.unique_scratch(n_cap))
    M = int(d_n.item())
    return out.cpu().numpy(), inv.cpu().numpy(), M, h.read_status()


def check_unique(h, rows, ts=0, fp=True):
    C, inv, M, st = unique(h, rows, ts, fp=fp)
    ref_rows = cref.floor_rows(rows) if fp else rows
    rc, ri = cref.unique_rows(ref_rows, ts)
    assert st == 0
    assert M == rc.shape[0] and np.array_equal(C[:M], rc) and np.array_equal(inv, ri)
    return rc


def random_rows(n, side, batches, seed):
    rng = np.random.default_rng(seed)
    return np.c_[rng.integers(0, batches, n), rng.integers(-side, side, (n, 3))].astype(np.int64)


# ---------------------------------------------------------------------------------------------------------
# lb2_unique_build
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 3 * 2048 + 1, 1_000_003])
def test_unique_build_scan_sizes(n):
    """first-occurrence rows and inverse across 1 .. 489 scan blocks, fp32 level-0 input and int32 stride levels"""
    h = H()
    rows = random_rows(n, max(2, int(round(0.45 * n ** (1 / 3)))), 3, n)       # about half the rows repeat a voxel
    C = check_unique(h, rows.astype(np.float32))
    check_unique(h, C, 2, fp=False)
    check_unique(h, C, 16, fp=False)


def test_unique_build_at_the_row_limit():
    """4 194 304 rows (2048 scan blocks): all distinct, all one voxel; one row more is refused"""
    h = H()
    n = 4 * 1024 * 1024
    rng = np.random.default_rng(0)
    i = rng.permutation(n)
    rows = np.c_[i % 3, (i // 3) % 160 - 80, (i // 480) % 160 - 80, i // 76800 - 27]
    C, inv, M, st = unique(h, rows.astype(np.int32), fp=False)
    assert st == 0 and M == n and np.array_equal(C, rows) and np.array_equal(inv, np.arange(n))
    same = np.tile(np.array([[2, -5, 7, 131071]]), (n, 1))
    C, inv, M, st = unique(h, same.astype(np.float32))
    assert st == 0 and M == 1 and C[0].tolist() == [2, -5, 7, 131071] and not inv.any()
    from lidiff_b200._lib import _ptr
    grid, buf = h.new_grid(16), torch.zeros(8, dtype=torch.int32, device=DEV)     # the row limit is checked first
    rc = h.dll.lb2_unique_build(h.hp, h._stream(), None, _ptr(buf), None, n + 1, 0, h._grid(grid), _ptr(buf), None, _ptr(buf), _ptr(buf))
    assert rc == -1, "n_cap above 4M rows must be refused (LB2_ERR_ARG)"


def test_unique_build_ignores_rows_past_the_live_count():
    """d_nin < n_cap: rows past the live count, out-of-range and NaN ones included, neither appear nor raise the status bit"""
    h = H()
    n_cap, n = 10_000, 6_001
    rows = random_rows(n_cap, 8, 2, 3).astype(np.float32)
    rows[n::7] = [5000, 1e6, -1e6, np.nan]
    rows[n + 1::7, 1] = np.inf
    rows[n + 2::7, 2] = LO - 1
    C, inv, M, st = unique(h, rows, n=n)
    rc, ri = cref.unique_rows(cref.floor_rows(rows[:n]))
    assert st == 0, "rows past the live count must not raise the status bit"
    assert M == rc.shape[0] and np.array_equal(C[:M], rc) and np.array_equal(inv[:n], ri)
    assert (inv[n:] == -7).all() and (C[M:] == 77).all(), "nothing is written past the live rows"


# ---------------------------------------------------------------------------------------------------------
# whole geometries: every level, map, mask, pair count and row order
# ---------------------------------------------------------------------------------------------------------
def check_geometry(g, coords, n):
    """engine Geometry built from coords (n, 4) fp32 against the restatement, levels 0..4 and all 13 maps"""
    N = g.n_cap
    lv, inv = [], []
    rc, ri = cref.unique_rows(cref.floor_rows(coords[:n]))
    lv.append(rc)
    inv.append(ri)
    for l in range(1, g.levels):
        rc, ri = cref.unique_rows(lv[-1], 1 << l)
        lv.append(rc)
        inv.append(ri)
    sizes = g.sizes()
    pairs = g.pairs.cpu().numpy()
    for l in range(g.levels):
        M = lv[l].shape[0]
        assert sizes[l] == M, ("rows", l)
        assert np.array_equal(g.C[l][:M].cpu().numpy(), lv[l]), ("coords", l)
        assert np.array_equal(g.inv[l][:inv[l].shape[0]].cpu().numpy(), inv[l]), ("inverse", l)
    maps = [(g.nbr3[l], g.perm3[l], lv[l], lv[l], 3, 1 << l, l, l) for l in range(g.levels)]
    maps += [(g.nbr_dn[l], g.perm_dn[l], lv[l - 1], lv[l], 2, 1 << (l - 1), 4 + l, l) for l in range(1, g.levels)]
    if g.nbr_up is not None:
        maps += [(g.nbr_up[l], g.perm_up[l], lv[l + 1], lv[l], 2, -(1 << l), 9 + l, l) for l in range(g.levels - 1)]
    for nbr, perm, cin, cout, ks, step, slot, l in maps:
        ref, mask, pc = cref.kernel_map(cin, cout, ks, step, N)
        what = (ks, step, l)
        assert np.array_equal(nbr.cpu().numpy(), ref), ("table",) + what
        assert np.array_equal(g.mask_of[nbr.data_ptr()].cpu().numpy().view(np.uint32), mask), ("row mask",) + what
        assert pairs[slot] == pc, ("pair count",) + what
        M = cout.shape[0]
        morton = ks == 3 and l in g.morton_levels
        want = cref.row_order(mask[:M], ks ** 3, cout if morton else None, l)
        assert np.array_equal(perm[:M].cpu().numpy(), want), ("row order",) + what
        b = cout[:, 0]
        hit = ref[:, :M] >= 0
        assert (cin[ref[:, :M][hit], 0] == np.broadcast_to(b, ref[:, :M].shape)[hit]).all(), ("a pair joins two batches",) + what


def build_geometry(h, coords, n_cap):
    from lidiff_b200.engine import Geometry
    g = Geometry(h, n_cap)
    g.build(f32(coords), coords.shape[0])
    torch.cuda.synchronize()
    assert h.read_status() == 0
    return g


def test_all_1024_batches_stay_apart():
    """the same 150 points in each of the 1024 batches: no voxel merges and no map pair joins across batches, at any level"""
    h = H()
    rng = np.random.default_rng(5)
    xyz = rng.integers(-40, 40, (150, 3))
    coords = np.c_[np.repeat(np.arange(1024), 150), np.tile(xyz, (1024, 1))].astype(np.float32)
    g = build_geometry(h, coords, coords.shape[0])
    assert g.sizes()[0] == 1024 * np.unique(xyz, axis=0).shape[0]
    check_geometry(g, coords, coords.shape[0])


def test_maps_at_the_key_range_limits():
    """rows at and next to -131072, -131071 and 131071 on every axis, batches 0 and 1023: every level and map equals the
    restatement (neighbours beyond the limit are misses, nothing wraps)"""
    h = H()
    near = np.array([LO, LO + 1, LO + 2, LO + 5, LO + 16, HI - 16, HI - 5, HI - 1, HI, 0])
    g3 = np.stack(np.meshgrid(near, near, near, indexing="ij"), -1).reshape(-1, 3)
    coords = np.concatenate([np.c_[np.zeros(len(g3)), g3], np.c_[np.full(len(g3), 1023), g3[::-1]]]).astype(np.float32)
    g = build_geometry(h, coords, coords.shape[0] + 100)
    check_geometry(g, coords, coords.shape[0])


def test_maps_at_scale():
    """500k points in 3 batches, fewer live rows than the capacity: every table, mask, pair count and row order (the restatement
    takes most of the time; the radix sort past 512 blocks is tested on its own below)"""
    h = H()
    rng = np.random.default_rng(7)
    n = 500_000
    pts = rng.standard_normal((n, 3)) * np.array([30.0, 30.0, 3.0])
    coords = np.c_[np.sort(rng.integers(0, 3, n)), np.round(pts / 0.05)].astype(np.float32)
    g = build_geometry(h, coords, n + 4099)
    check_geometry(g, coords, n)


# ---------------------------------------------------------------------------------------------------------
# the status bit
# ---------------------------------------------------------------------------------------------------------
BAD_F = [[-1, 0, 0, 0], [1024, 0, 0, 0], [0, 131072, 0, 0], [0, 0, -131073, 0], [0, 0, 0, np.inf], [0, -np.inf, 0, 0],
         [0, 3e9, 0, 0], [0, 0, -3e9, 0], [0, 0, 0, np.nan], [np.nan, 0, 0, 0], [0, np.nan, 0, 0]]
BAD_I = [[-1, 0, 0, 0], [1024, 0, 0, 0], [0, 131072, 0, 0], [0, 0, -131073, 0], [0, 0, 0, 2 ** 31 - 1], [0, -2 ** 31, 0, 0]]
GOOD = [[0, LO, LO, LO], [1023, HI, HI, HI], [0, LO, HI, 0], [1023.99, HI + 0.99, LO, 0.5]]


def test_status_bit_is_raised_by_exactly_the_out_of_range_rows():
    """each case alone between two status reads, through in_f and (where it has an int32 form) in_i"""
    from lidiff_b200 import me
    h = H()
    base = random_rows(300, 10, 2, 1).astype(np.float32)
    h.read_status()                                             # clear whatever an earlier test left
    for row in GOOD:
        for fp in (True, False):
            r = np.concatenate([base, [row]])
            _, _, _, st = unique(h, r if fp else cref.floor_rows(r).astype(np.int32), fp=fp)
            assert st == 0, (row, fp)
    for row in BAD_F:
        r = np.concatenate([base, [row]]).astype(np.float32)
        assert cref.flagged(in_f=r)[-1]
        _, _, _, st = unique(h, r)
        assert st == 1, ("in_f", row)
        with pytest.raises(RuntimeError, match="key range"):
            me.TensorField(torch.zeros(r.shape[0], 3, device=DEV), f32(r)).sparse()
        assert h.read_status() == 0
    for row in BAD_I:
        r = np.concatenate([base.astype(np.int64), [row]])
        _, _, _, st = unique(h, r.astype(np.int32), fp=False)
        assert st == 1, ("in_i", row)
    me.TensorField(torch.zeros(len(GOOD), 3, device=DEV), f32(GOOD)).sparse()


# ---------------------------------------------------------------------------------------------------------
# lb2_row_order
# ---------------------------------------------------------------------------------------------------------
def row_order(h, mask, kvol, coords=None, shift=0, n=None):
    N = mask.shape[0]
    perm = torch.full((N,), -3, dtype=torch.int32, device=DEV)
    scratch = torch.zeros(h.row_order_scratch_bytes(N), dtype=torch.uint8, device=DEV)
    h.row_order(i32(mask.view(np.int32)), None if n is None else i32([n]), N, kvol, perm, scratch,
                None if coords is None else i32(coords), shift)
    return perm.cpu().numpy()


def test_row_order_equals_the_stable_sort_at_scale():
    """1.1M rows (538 radix blocks), masks from a small pool so that many rows share a key: kvol 27 with and without
    coordinates, kvol 8, and a live count below the capacity"""
    h = H()
    rng = np.random.default_rng(11)
    N = 1_100_000
    c = 1 << 13
    pool27 = np.array([c, c | 1, c | 2, c | (1 << 26), c | 3, c | 0x5555, c | (0x7FFFFFF ^ c), 0x7FFFFFF, c | (1 << 20) | 1], np.uint32)
    pool8 = np.array([0, 1, 2, 0x81, 0xFF, 0x10, 0x3C], np.uint32)
    m27, m8 = pool27[rng.integers(0, len(pool27), N)], pool8[rng.integers(0, len(pool8), N)]
    coords = np.c_[np.zeros(N, int), rng.integers(-3000, 3000, (N, 3)) * 4]
    assert np.array_equal(row_order(h, m27, 27), cref.row_order(m27, 27))
    assert np.array_equal(row_order(h, m27, 27, coords, 2), cref.row_order(m27, 27, coords, 2))
    assert np.array_equal(row_order(h, m8, 8), cref.row_order(m8, 8))
    n = 777_777
    got = row_order(h, m27, 27, coords, 2, n=n)
    assert np.array_equal(got[:n], cref.row_order(m27[:n], 27, coords[:n], 2)) and (got[n:] == -3).all()
    got = row_order(h, m8, 8, n=n)
    assert np.array_equal(got[:n], cref.row_order(m8[:n], 8)) and (got[n:] == -3).all()


@pytest.mark.parametrize("kvol", [27, 8])
def test_row_order_keeps_equal_masks_in_index_order(kvol):
    h = H()
    mask = np.full(10_000, (1 << 13) | 5 if kvol == 27 else 5, np.uint32)
    assert np.array_equal(row_order(h, mask, kvol), np.arange(10_000))
    if kvol == 27:
        assert np.array_equal(row_order(h, mask, kvol, np.zeros((10_000, 4), int)), np.arange(10_000))


# ---------------------------------------------------------------------------------------------------------
# lb2_voxel_mean
# ---------------------------------------------------------------------------------------------------------
def voxel_mean(h, feats, inv, m, m_cap=None):
    m_cap = m if m_cap is None else m_cap
    n, c = feats.shape
    out = torch.full((m_cap, c), 5.0, device=DEV)
    h.voxel_mean(f32(feats), i32(inv), n, c, i32([m]), m_cap, out, h.voxel_mean_scratch(m_cap, c))
    return out.cpu().numpy()


@pytest.mark.parametrize("name", cref.VOXEL_MEAN_CASES)
def test_voxel_mean_meets_the_bound_and_the_equality_rule(name):
    h = H()
    feats, inv, m = cref.voxel_mean_case(name)
    got = voxel_mean(h, feats, inv, m, m + 37)
    assert (got[m:] == 0).all() and not np.signbit(got[m:]).any(), "rows past the live count stay 0"
    bb, eb, n_eq = cref.check_voxel_mean(feats, inv, m, got[:m])
    print(f"{name}: {n_eq} of {bb.size} means required equal to RN32(mean); bound violations {int(bb.sum())}, "
          f"equality violations {int(eb.sum())}")
    assert not bb.any(), np.argwhere(bb)[:8]
    assert not eb.any(), np.argwhere(eb)[:8]


def test_voxel_mean_does_not_depend_on_the_order_of_the_points():
    h = H()
    rng = np.random.default_rng(3)
    n, m = 1_000_000, 120_000
    inv = rng.integers(0, m, n).astype(np.int32)
    inv[:m] = np.arange(m)
    feats = (rng.standard_normal((n, 3)) * 10.0 ** rng.uniform(-3, 3, (n, 1))).astype(np.float32)
    ref = voxel_mean(h, feats, inv, m)
    bb, eb, _ = cref.check_voxel_mean(feats, inv, m, ref)
    assert not bb.any() and not eb.any()
    for s in range(8):
        p = np.random.default_rng(100 + s).permutation(n)
        assert np.array_equal(voxel_mean(h, feats[p], inv[p], m).view(np.int32), ref.view(np.int32)), s


# ---------------------------------------------------------------------------------------------------------
# nearest key voxel: the shared-memory table past its capacity and shells across the key-range limit
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nk", [8192, 8193])
def test_nn_table_at_and_past_its_capacity_equals_brute_force(nk):
    h = H()
    rng = np.random.default_rng(nk)
    cells = np.unique(rng.integers(-60, 60, (3 * nk, 3)), axis=0)
    cells = cells[rng.permutation(cells.shape[0])][: nk - 8] * 16
    edge = np.array([[LO, 0, 0], [LO, LO, LO], [HI - 15, 0, 0], [HI - 15, HI - 15, HI - 15], [0, LO, HI - 15],
                     [LO + 16, 0, 0], [0, HI - 31, 0], [LO, HI - 15, 0]])       # lattice cells next to both limits
    kxyz = np.concatenate([cells, edge])
    keys = np.c_[np.zeros(nk, int), kxyz]
    assert np.unique(keys, axis=0).shape[0] == nk
    kc, _, M, st = unique(h, keys.astype(np.int32), fp=False)
    assert st == 0 and M == nk
    near = kxyz[rng.integers(0, nk, 20_000)] + rng.integers(-40, 40, (20_000, 3))
    limit = np.concatenate([np.c_[rng.integers(LO, LO + 40, (3000, 1)), rng.integers(-40, 40, (3000, 2))],
                            np.c_[rng.integers(HI - 40, HI + 1, (3000, 1)), rng.integers(HI - 40, HI + 1, (3000, 2))],
                            np.c_[rng.integers(LO, LO + 40, (3000, 2)), rng.integers(LO, LO + 40, (3000, 1))]])
    q = np.c_[np.zeros(29_000, int), np.clip(np.concatenate([near, limit]), LO, HI)]
    qd, kd = i32(q), i32(kc)
    a, b, t = (torch.empty(q.shape[0], dtype=torch.int32, device=DEV) for _ in range(3))
    h.nn_match(qd, None, q.shape[0], kd, None, nk, 0, a)
    tab = h.nn_table(kd, None, nk)
    h.nn_match_table(qd, None, q.shape[0], kd, None, nk, tab, 16, 4, t)
    assert torch.equal(a, t), "shared-memory table"
    grid = h.new_grid(nk)
    h.unique_build(None, kd, None, nk, 0, grid, torch.empty_like(kd), None, i32([0]), h.unique_scratch(nk))
    h.nn_match_grid(qd, None, q.shape[0], kd, None, nk, grid, 16, 4, b)
    assert torch.equal(a, b), "hash-grid shell search"
