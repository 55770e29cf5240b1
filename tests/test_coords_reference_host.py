"""The coordinate manager's restatement (tests/coords_reference.py) checked without a GPU: hand-checkable answers for unique rows,
the key range, kernel maps and row order; the voxel-mean bound holds for a host emulation of the kernel's fixed-point arithmetic
and rejects a voxel mean accumulated in fp32 in shuffled order (so the GPU test of lb2_voxel_mean has teeth)."""
import numpy as np
import pytest
import torch

import coords_reference as cref
import fake_backend
from oracle import me_cpu as ome


def test_unique_rows_two_by_two_block_negative_floors_and_strides():
    rows = np.array([[0, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 1, 1, 1], [0, -1, -1, -1], [0, 0, 0, 0],
                     [0, -2, -3, -4]])
    C, inv = cref.unique_rows(rows)
    assert C.tolist() == [[0, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 1, 1, 1], [0, -1, -1, -1], [0, -2, -3, -4]]
    assert inv.tolist() == [0, 1, 2, 1, 3, 4, 0, 5]
    C2, inv2 = cref.unique_rows(rows, 2)                 # true floor: -1 -> -2, -3 -> -4
    assert C2.tolist() == [[0, 0, 0, 0], [0, -2, -2, -2], [0, -2, -4, -4]]
    assert inv2.tolist() == [0, 0, 0, 0, 0, 1, 0, 2]
    f = np.array([[0, 0.5, -0.5, -1.0], [0, 0.99, -0.01, -1.5]], np.float32)
    assert cref.floor_rows(f).tolist() == [[0, 0, -1, -1], [0, 0, -1, -2]]


def test_two_batches_with_the_same_xyz_stay_apart():
    xyz = np.array([[5, 5, 5], [6, 5, 5], [5, 5, 5]])
    rows = np.concatenate([np.c_[np.zeros(3, int), xyz], np.c_[np.ones(3, int), xyz]])
    C, inv = cref.unique_rows(rows)
    assert C.tolist() == [[0, 5, 5, 5], [0, 6, 5, 5], [1, 5, 5, 5], [1, 6, 5, 5]]
    assert inv.tolist() == [0, 1, 0, 2, 3, 2]
    nbr, mask, pairs = cref.kernel_map(C, C, 3, 1)
    assert nbr[13].tolist() == [0, 1, 2, 3] and nbr[14].tolist() == [1, -1, 3, -1] and nbr[12].tolist() == [-1, 0, -1, 2]
    assert pairs == 8 and mask.tolist() == [(1 << 13) | (1 << 14), (1 << 13) | (1 << 12)] * 2


def test_key_range_limits():
    lo, hi = cref.AXIS_MIN, cref.AXIS_MAX
    assert (lo, hi) == (-131072, 131071) and (ome.AXIS_OFF == -lo)
    rows = np.array([[0, lo, 0, 0], [0, hi, hi, hi], [1023, lo, lo, lo], [0, lo - 1, 0, 0], [0, 0, hi + 1, 0], [-1, 0, 0, 0],
                     [1024, 0, 0, 0]])
    assert cref.flagged(in_i=rows).tolist() == [False] * 3 + [True] * 4
    assert ome.in_key_range(rows[:, 1:]).tolist() == [True] * 3 + [False, False, True, True]
    f = np.array([[0, lo, hi, 0], [0, np.nan, 0, 0], [np.nan, 0, 0, 0], [0, np.inf, 0, 0], [0, 0, -np.inf, 0], [0, 3e9, 0, 0],
                  [0, -3e9, 0, 0], [0, hi + 0.99, 0, 0], [0, lo - 0.01, 0, 0], [1023.9, 0, 0, 0]], np.float32)
    assert cref.flagged(in_f=f).tolist() == [False, True, True, True, True, True, True, False, True, False]
    assert cref.floor_rows(f)[1].tolist() == [0, 0, 0, 0] and cref.floor_rows(f)[3, 1] == cref.I32_MAX
    # a row at the lower limit stays in range at every stride level (the range is closed under the floor to 2^l)
    for ts in (2, 4, 8, 16):
        assert cref.floor_to(np.array([[0, lo + ts - 1, lo + 1, lo]]), ts)[0, 1:].tolist() == [lo, lo, lo]
    # neighbours across the limit are misses, never wrapped
    C = np.array([[0, lo, 0, 0], [0, hi, 0, 0], [0, lo + 1, 0, 0]])
    nbr, mask, pairs = cref.kernel_map(C, C, 3, 1)
    assert nbr[12].tolist() == [-1, -1, 0] and nbr[14].tolist() == [2, -1, -1] and pairs == 5
    nbr, _, _ = cref.kernel_map(C, C[:1], 2, -1)          # transposed: offsets 0 and -1 on each axis
    assert nbr[:, 0].tolist() == [0] + [-1] * 7


def test_kernel_map_dead_rows_and_oracle_pair_sets():
    rng = np.random.default_rng(0)
    rows = np.c_[rng.integers(0, 2, 3000), rng.integers(-6, 6, (3000, 3))]
    C, _ = cref.unique_rows(rows)
    nbr, mask, pairs = cref.kernel_map(C, C[:100], 3, 1, n_cap=130)
    assert (nbr[:, 100:] == -1).all() and (mask[100:] == 0).all()
    geom = ome.Geometry(C, np.arange(C.shape[0]))
    ref = cref.kernel_map(C, C, 3, 1)[0]
    for k, (i, o) in enumerate(geom.kernel_map(1, 3, 1)):
        assert set(zip(i.tolist(), o.tolist())) == set(zip(ref[k][ref[k] >= 0].tolist(), np.nonzero(ref[k] >= 0)[0].tolist()))


def test_row_order_known_answers():
    c = 1 << 13
    mask = np.array([c | 1, c, c | 3, c, c | 1, c | (1 << 26), c | 5], np.uint32)
    # keys: [c|1] -> 1, [c] -> 0, [c|3] -> 2^26|3, [c|2^26] -> 2^25, [c|5] -> 2^26|5
    assert cref.row_order(mask, 27).tolist() == [1, 3, 0, 4, 5, 2, 6]
    assert cref.row_order(np.array([3, 1, 3, 0, 0x103], np.uint32), 8).tolist() == [3, 1, 0, 2, 4]
    coords = np.array([[0, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 0], [0, 0, 1, 0], [0, 0, 0, 0], [0, 2, 0, 0], [0, 0, 0, 0]])
    same = np.full(7, c, np.uint32)
    assert cref.row_order(same, 27, coords).tolist() == [0, 2, 4, 6, 1, 3, 5]
    assert cref.row_order(same, 27, coords * 2, shift=1).tolist() == [0, 2, 4, 6, 1, 3, 5]
    assert cref.morton(np.array([[0, 512, 513, -1]]), 0).tolist() == [(1 << 1) | (0x1249249 << 2)]     # 9 bits per axis, wrapped


def test_voxel_mean_known_answers():
    feats = np.array([[1.0, 3.0], [2.0, -3.0], [4.0, 0.0], [np.nan, 0.0]], np.float32)
    inv = np.array([0, 0, 1, 2])
    got = np.array([[1.5, 0.0], [4.0, 0.0], [np.nan, 0.0], [np.nan, np.nan]], np.float32)     # row 3: no members
    bb, eb, n_eq = cref.check_voxel_mean(feats, inv, 4, got)
    assert not bb.any() and not eb.any() and n_eq == 2
    bad = got.copy()
    bad[0, 0] = np.nextafter(np.float32(1.5), np.float32(2))
    assert cref.check_voxel_mean(feats, inv, 4, bad)[1][0, 0], "one ulp off an exactly representable mean"
    bad = got.copy()
    bad[1, 1] = -0.0
    assert cref.check_voxel_mean(feats, inv, 4, bad)[0][1, 1], "an all-zero row is +0"


@pytest.mark.parametrize("name", cref.VOXEL_MEAN_CASES)
def test_fixed_point_emulation_meets_the_bound_and_the_equality_rule(name):
    feats, inv, m = cref.voxel_mean_case(name)
    got = cref.emulate_voxel_mean(feats, inv, m)
    bb, eb, n_eq = cref.check_voxel_mean(feats, inv, m, got)
    print(f"{name}: {n_eq} of {got.size} means required equal to RN32(mean)")
    assert not bb.any() and not eb.any()
    if name.startswith("random"):
        assert n_eq >= 0.9 * got.size, "the equality rule should apply almost everywhere"
    perm = np.random.default_rng(1).permutation(inv.shape[0])
    assert np.array_equal(cref.emulate_voxel_mean(feats[perm], inv[perm], m).view(np.int32), got.view(np.int32))


@pytest.mark.parametrize("name", cref.CANCELLATION_CASES)
def test_fp32_accumulation_in_shuffled_order_fails_the_bound(name):
    """the fp32 index_add_ form (the fake backend's, ME's) loses the small remainders of cancelling members"""
    feats, inv, m = cref.voxel_mean_case(name)
    perm = np.random.default_rng(2).permutation(inv.shape[0])
    f, i = torch.from_numpy(feats[perm]), torch.from_numpy(inv[perm]).long()
    sums = torch.zeros(m, feats.shape[1]).index_add_(0, i, f)
    got = (sums / torch.bincount(i, minlength=m).float()[:, None]).numpy()
    bb, eb, _ = cref.check_voxel_mean(feats, inv, m, got)
    print(f"{name}: fp32 accumulation violates the bound in {int(bb.sum())} of {bb.size} means")
    assert bb.sum() >= 2


def test_fake_backend_raises_the_status_bit_for_the_same_rows(monkeypatch):
    h = fake_backend.install(monkeypatch)
    from lidiff_b200 import me
    ok = torch.tensor([[0, -131072, 131071, 0], [1023, 5, 5, 5]], dtype=torch.float32)
    for bad_row, want in ((None, 0), ([0, np.nan, 0, 0], 1), ([np.nan, 0, 0, 0], 1), ([0, 131072, 0, 0], 1),
                          ([0, 0, -131073, 0], 1), ([1024, 0, 0, 0], 1), ([-1, 0, 0, 0], 1), ([0, np.inf, 0, 0], 1), ([0, -3e9, 0, 0], 1)):
        C = ok if bad_row is None else torch.cat([ok, torch.tensor([bad_row], dtype=torch.float32)])
        F = torch.zeros(C.shape[0], 3)
        if want:
            with pytest.raises(RuntimeError, match="key range"):
                me.TensorField(F, C).sparse()
        else:
            me.TensorField(F, C).sparse()
        assert h.read_status() == 0, "me.py reads (and clears) the status word behind the level-0 build"
