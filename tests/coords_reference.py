"""TEST INFRASTRUCTURE: a plain numpy restatement of the coordinate manager's contract (include/lidiff_b200.h,
lidiff_b200/csrc/coords.cu), integer arithmetic only, for bit-exact comparison with the CUDA kernels.

  key range        batch in [0, 1023], every axis in [-131072, 131071]; an fp32 input row is floored and converted like
                   the kernel's (int)floorf: NaN -> 0, +-inf and huge values saturate to INT_MIN / INT_MAX.  A row whose
                   converted value is outside the range, or that has a NaN component, raises status bit 0.
  unique rows      first-occurrence order, inverse[i] = output row of input row i; ts_floor > 0 floors the axes to multiples
                   of ts_floor (true floor for negatives) first.
  kernel maps      nbr[k][o] = input row at out[o] + offset_k * step or -1 (a neighbour outside the key range is a miss),
                   row_mask[o] bit k <=> nbr[k][o] >= 0, pair_count = number of hits; rows o in [n, n_cap) get -1 / 0.
  row order        the stable sort of lb2_row_order: 8-bit masks, or the 27-bit key [>= 2 off-centre | mask without centre]
                   with, if coordinates are given, the Morton code of (x, y, z) >> shift (9 bits per axis, wrapped) next,
                   then the row index.
  voxel mean       error bound and equality rule of the fixed-point mean (see check_voxel_mean).
"""
import numpy as np

AXIS_MIN, AXIS_MAX = -(1 << 17), (1 << 17) - 1
BATCH_MAX = 1023
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1


# ---------------------------------------------------------------------------------------------------------
# rows and the key range
# ---------------------------------------------------------------------------------------------------------
def floor_rows(in_f):
    """(n, 4) fp32 -> int64 rows as the kernel converts them: floor, NaN -> 0, saturation to int32"""
    f = np.floor(np.asarray(in_f, dtype=np.float32).astype(np.float64))
    f = np.where(np.isnan(f), 0.0, f)
    return np.clip(f, I32_MIN, I32_MAX).astype(np.int64)


def in_range(rows):
    """(n, 4) integer rows -> bool (n,): batch and axes inside the key range"""
    rows = np.asarray(rows, dtype=np.int64)
    return ((rows[:, 0] >= 0) & (rows[:, 0] <= BATCH_MAX)
            & ((rows[:, 1:] >= AXIS_MIN) & (rows[:, 1:] <= AXIS_MAX)).all(1))


def flagged(in_f=None, in_i=None):
    """the input rows that raise status bit 0 (bool (n,))"""
    if in_f is not None:
        in_f = np.asarray(in_f, dtype=np.float32)
        return ~in_range(floor_rows(in_f)) | np.isnan(in_f).any(1)
    return ~in_range(in_i)


def pack(rows):
    rows = np.asarray(rows, dtype=np.int64)
    assert in_range(rows).all()
    return (rows[:, 0] << 54) | ((rows[:, 1] - AXIS_MIN) << 36) | ((rows[:, 2] - AXIS_MIN) << 18) | (rows[:, 3] - AXIS_MIN)


def floor_to(rows, ts):
    rows = np.asarray(rows, dtype=np.int64).copy()
    if ts > 0:
        rows[:, 1:] = np.floor_divide(rows[:, 1:], ts) * ts
    return rows


def unique_rows(rows, ts_floor=0):
    """(coords (M, 4) int32, inverse (n,) int32) in first-occurrence order"""
    rows = floor_to(rows, ts_floor)
    if rows.shape[0] == 0:
        return np.zeros((0, 4), np.int32), np.zeros(0, np.int32)
    _, first, inv = np.unique(pack(rows), return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(order.shape[0])
    return rows[first[order]].astype(np.int32), rank[inv.reshape(-1)].astype(np.int32)


# ---------------------------------------------------------------------------------------------------------
# kernel maps
# ---------------------------------------------------------------------------------------------------------
def offsets(ks):
    """(ks^3, 3) offsets in units of `step`, k = kx + ks*ky + ks*ks*kz; odd ks centred"""
    r = np.arange(ks)
    kz, ky, kx = np.meshgrid(r, r, r, indexing="ij")
    o = np.stack([kx.reshape(-1), ky.reshape(-1), kz.reshape(-1)], 1).astype(np.int64)
    return o - ks // 2 if ks % 2 else o


def kernel_map(in_coords, out_coords, ks, step, n_cap=None):
    """-> nbr (ks^3, n_cap) int32, row_mask (n_cap,) uint32, pair_count; `in_coords` are the rows of the grid (row id =
    index), the first len(out_coords) rows of the table are live"""
    in_coords, out_coords = np.asarray(in_coords, np.int64), np.asarray(out_coords, np.int64)
    n = out_coords.shape[0]
    n_cap = n if n_cap is None else n_cap
    keys = pack(in_coords)
    order = np.argsort(keys, kind="stable")
    skeys = keys[order]
    K = ks ** 3
    nbr = np.full((K, n_cap), -1, np.int32)
    mask = np.zeros(n_cap, np.uint32)
    for k, off in enumerate(offsets(ks) * step):
        q = out_coords.copy()
        q[:, 1:] += off[None, :]
        ok = in_range(q)
        qk = pack(np.where(ok[:, None], q, 0))
        pos = np.minimum(np.searchsorted(skeys, qk), max(skeys.shape[0] - 1, 0))
        hit = ok & (skeys[pos] == qk) if skeys.shape[0] else np.zeros(n, bool)
        nbr[k, :n] = np.where(hit, order[pos], -1)
        mask[:n] |= hit.astype(np.uint32) << np.uint32(k)
    return nbr, mask, int((nbr >= 0).sum())


# ---------------------------------------------------------------------------------------------------------
# row order
# ---------------------------------------------------------------------------------------------------------
def _popcount(v):
    v = np.asarray(v, np.uint64)
    c = np.zeros(v.shape, np.int64)
    for b in range(32):
        c += ((v >> np.uint64(b)) & np.uint64(1)).astype(np.int64)
    return c


def row_order_key(mask, kvol):
    m = np.asarray(mask).astype(np.int64) & 0xFFFFFFFF
    if kvol <= 8:
        return m & 0xFF
    extras = m & ~(1 << 13)
    key = ((_popcount(extras) >= 2).astype(np.int64) << 26) | ((m >> 14) << 13) | (m & 0x1FFF)
    return key & ((1 << 27) - 1)                         # 3 passes of 9 bits


def _part9(v):
    v = v & 0x1FF
    out = np.zeros_like(v)
    for b in range(9):
        out |= ((v >> b) & 1) << (3 * b)
    return out


def morton(coords, shift):
    c = np.asarray(coords, np.int64)
    return _part9(c[:, 1] >> shift) | (_part9(c[:, 2] >> shift) << 1) | (_part9(c[:, 3] >> shift) << 2)


def row_order(mask, kvol, coords=None, shift=0):
    """the permutation lb2_row_order writes for the live rows `mask` (and their `coords`)"""
    key = row_order_key(mask, kvol)
    if coords is None or kvol != 27:
        return np.argsort(key, kind="stable").astype(np.int32)
    return np.lexsort((morton(coords, shift), key)).astype(np.int32)      # last key primary; ties in index order


# ---------------------------------------------------------------------------------------------------------
# voxel mean
# ---------------------------------------------------------------------------------------------------------
def _ulp32(x):
    """fp32 ulp at |x| (subnormal spacing below 2^-126)"""
    e = np.where(x == 0, -125, np.frexp(np.abs(x))[1])
    return np.ldexp(1.0, np.maximum(e, -125) - 24)


def check_voxel_mean(feats, inverse, m, got):
    """Check `got` (m, c) fp32 against the contract of lb2_voxel_mean for the members feats (n, c) fp32 of rows inverse (n,).

    For each (row, channel) with n members, largest magnitude in [2^(e-1), 2^e), s = 61 - e - bitlen(n) and exact mean mu:
        |got - mu| <= ulp32(mu)/2 + 2^-(s+1) + 2^-50 |mu|                                        (bound)
    and got == RN32(mu) wherever mu is farther than 2^-(s+1) + 2^-50 |mu| from every fp32 rounding midpoint (equality).
    A row with a NaN or +-inf member, or with no member, is NaN; a row whose members are all zero is +0.

    mu is computed from two exact int64 limb sums per (row, channel) (each member split at 2^(e-w) and rounded at 2^(e-2w),
    w = 62 - bitlen(max n)), then in fp64: its error eta <= 2^-51 |mu| + 2^(e-w-50), far below 2^-(s+1), is added to both
    margins.  Returns (bound_violations, equality_violations, n_equality_checked); the violation arrays are bool (m, c)."""
    F = np.asarray(feats, np.float32)
    inv = np.asarray(inverse, np.int64)
    got = np.asarray(got, np.float32)
    c = F.shape[1]
    cnt = np.bincount(inv, minlength=m)[:m]
    order = np.argsort(inv, kind="stable")
    F, inv = F[order].astype(np.float64), inv[order]
    live = np.nonzero(cnt)[0]
    starts = np.concatenate([[0], np.cumsum(cnt)])[live]
    finite = np.isfinite(F)
    nonfinite = np.zeros((m, c), bool)
    nonfinite[live] = np.logical_or.reduceat(~finite, starts, axis=0)
    F = np.where(finite, F, 0.0)
    maxabs = np.zeros((m, c))
    maxabs[live] = np.maximum.reduceat(np.abs(F), starts, axis=0)
    e = np.frexp(maxabs)[1]                                          # maxabs < 2^e (0 for maxabs = 0)
    w = 62 - max(int(cnt.max()).bit_length(), 1)
    E = e[inv]
    u1, u2 = np.ldexp(1.0, E - w), np.ldexp(1.0, E - 2 * w)
    hi = np.floor(F / u1)
    lo = np.rint((F - hi * u1) / u2)
    SH = np.zeros((m, c), np.int64)
    SL = np.zeros((m, c), np.int64)
    SH[live] = np.add.reduceat(hi.astype(np.int64), starts, axis=0)
    SL[live] = np.add.reduceat(lo.astype(np.int64), starts, axis=0)
    n = np.maximum(cnt, 1)[:, None].astype(np.float64)
    mu = (SH.astype(np.float64) * np.ldexp(1.0, e - w) + SL.astype(np.float64) * np.ldexp(1.0, e - 2 * w)) / n
    eta = np.ldexp(np.abs(mu), -51) + np.ldexp(1.0, e - w - 50)
    bl = np.array([int(v).bit_length() for v in np.maximum(cnt, 1)])[:, None]
    q = np.ldexp(1.0, e + bl - 62)                                   # 2^-(s+1)
    slack = q + np.ldexp(np.abs(mu) + eta, -50) + eta
    g = got.astype(np.float64)
    special = nonfinite | (cnt == 0)[:, None] | (maxabs == 0)
    with np.errstate(invalid="ignore", over="ignore"):
        bound_bad = ~(np.abs(g - mu) <= 0.5 * _ulp32(np.abs(mu) + eta) + slack)
        f = mu.astype(np.float32)
        half = 0.5 * _ulp32(f.astype(np.float64))
        lower = np.abs(f.astype(np.float64)) - 0.5 * _ulp32(np.nextafter(np.abs(f), np.float32(0)).astype(np.float64))
        upper = np.abs(f.astype(np.float64)) + half
        dist = np.minimum(np.abs(np.abs(mu) - lower), np.abs(upper - np.abs(mu)))
        need_eq = (dist > slack + eta) & ~special
        eq_bad = need_eq & (got.view(np.int32) != f.view(np.int32))
    want_nan = nonfinite | (cnt == 0)[:, None]
    zero = (maxabs == 0) & ~want_nan
    bound_bad = np.where(want_nan, ~np.isnan(got), np.where(zero, got.view(np.int32) != 0, bound_bad))
    eq_bad = eq_bad | (zero & (got.view(np.int32) != 0))
    return bound_bad, eq_bad, int(need_eq.sum())


def emulate_voxel_mean(feats, inverse, m):
    """the kernel's arithmetic on the host: per (row, channel) every member rounded to 2^-s (s = 61 - e - bitlen(n)), int64 sum,
    fp64 scale and division, one rounding to fp32 (a faithful implementation, for checking check_voxel_mean itself)"""
    F = np.asarray(feats, np.float32).astype(np.float64)
    inv = np.asarray(inverse, np.int64)
    c = F.shape[1]
    cnt = np.bincount(inv, minlength=m)[:m]
    maxabs = np.zeros((m, c))
    np.maximum.at(maxabs, inv, np.abs(F))
    e = np.frexp(maxabs)[1]
    bl = np.array([int(v).bit_length() for v in cnt])[:, None]
    s = 61 - e - bl
    q = np.rint(np.ldexp(np.where(np.isfinite(F), F, 0.0), s[inv])).astype(np.int64)
    S = np.zeros((m, c), np.int64)
    np.add.at(S, inv, q)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = (np.ldexp(S.astype(np.float64), -s) / cnt[:, None]).astype(np.float32)
    out[maxabs == 0] = 0.0
    out[~np.isfinite(maxabs) | (cnt == 0)[:, None]] = np.nan
    return out


# ---------------------------------------------------------------------------------------------------------
# voxel-mean cases (members feats (n, c) fp32, inverse (n,) int32, rows m), shared by the host and the GPU tests
# ---------------------------------------------------------------------------------------------------------
FMAX, FTINY = float(np.finfo(np.float32).max), 2.0 ** -149


def _voxels(groups):
    """list of member lists (each member a length-c sequence) -> (feats, inverse, m), members of a voxel interleaved with others"""
    rows, inv = [], []
    for v, g in enumerate(groups):
        rows += list(g)
        inv += [v] * len(g)
    feats, inv = np.asarray(rows, np.float32).reshape(len(inv), -1), np.asarray(inv, np.int32)
    perm = np.random.default_rng(len(inv)).permutation(len(inv))
    return feats[perm], inv[perm], len(groups)


def voxel_mean_case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("random_c"):                          # 1..5000 members per voxel, magnitudes over 12 decades
        c = int(name[len("random_c"):])
        V = {1: 400, 3: 300, 7: 150, 96: 16}[c]
        counts = np.minimum(np.exp(rng.uniform(0, np.log(5000), V)).astype(np.int64), 5000)
        counts[:3] = (1, 2, 5000)
        scale = 10.0 ** rng.uniform(-6, 6, (V, 1))
        centre = rng.standard_normal((V, c)) * 3
        inv = np.repeat(np.arange(V), counts)
        feats = ((centre[inv] + rng.standard_normal((inv.shape[0], c))) * scale[inv]).astype(np.float32)
        perm = rng.permutation(inv.shape[0])
        return feats[perm], inv[perm].astype(np.int32), V
    if name == "cancel":                                     # large members that cancel, a small remainder
        g = [[[1e8], [-1e8], [1e-3]], [[1e-3], [1e8], [-1e8]], [[3e7], [1.0], [-3e7], [1.0]], [[1e20], [7.0], [-1e20]]]
        for n in (100, 10_000):
            a = rng.standard_normal(n // 2) * 1e3
            g.append([[v] for v in np.concatenate([a, -a, [1e-2]])])
            b = (rng.standard_normal(n) * 10).astype(np.float32)
            g.append([[v] for v in np.concatenate([b, [-np.sum(b.astype(np.float64))]])])
        return _voxels(g)
    if name == "extremes":                                   # subnormal and FLT_MAX members, 30-decade mixes
        g = [[[FTINY]], [[FTINY], [FTINY], [FTINY]], [[FTINY], [-FTINY], [FTINY]], [[FTINY], [3 * FTINY]], [[FMAX]],
             [[FMAX], [FMAX], [FMAX]], [[FMAX], [-FMAX], [FTINY]], [[FMAX], [FMAX / 2], [-FMAX]], [[1e30], [-1e30], [1e-30]],
             [[1e30], [1e-30], [1e-30]], [[1e-30]] * 5, [[1e-30], [-3e-30], [2e-38]], [[0.0], [-0.0]], [[2.0 ** -126], [-FTINY]]]
        return _voxels(g)
    if name == "nonfinite":                                  # one NaN / inf member poisons its voxel, not the others
        g = [[[np.nan, 1.0], [2.0, 3.0]], [[np.inf, 1.0], [1.0, 1.0]], [[-np.inf, 1.0], [5.0, 1.0]], [[np.inf, 0.0], [-np.inf, 0.0]],
             [[1.0, 2.0], [3.0, 4.0]], [[FMAX, -np.nan]]]
        return _voxels(g)
    raise ValueError(name)


VOXEL_MEAN_CASES = ["random_c1", "random_c3", "random_c7", "random_c96", "cancel", "extremes", "nonfinite"]
CANCELLATION_CASES = ["cancel", "extremes"]
