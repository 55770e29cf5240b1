"""Host side of the offset split: the per-layer table, its LB2_OFFSET_SPLIT override and which convolutions it applies to."""
import pytest

from lidiff_b200.engine import OFFSET_RANGES, OFFSET_SPLIT_DEFAULT, offset_split_table, one_offset_per_group, split_level


def test_ranges_are_contiguous_and_cover_the_kernel():
    for G, rs in OFFSET_RANGES.items():
        assert len(rs) == G and rs[0][0] == 0 and rs[-1][1] == 27
        assert all(a[1] == b[0] and a[0] < a[1] for a, b in zip(rs, rs[1:]))


def test_table_and_override():
    assert offset_split_table("") == OFFSET_SPLIT_DEFAULT
    assert offset_split_table("3") == {k: 3 for k in OFFSET_SPLIT_DEFAULT}
    t = offset_split_table("stage4=2, up2=1")
    assert t["stage4"] == 2 and t["up2"] == 1 and t["up1"] == OFFSET_SPLIT_DEFAULT["up1"]
    with pytest.raises(ValueError):
        offset_split_table("up1=4")


def test_which_convs_split():
    assert split_level("stage4.1.net.0") == ("stage4", 4) and split_level("stage4.2.net.3") == ("stage4", 4)
    assert split_level("up1.1.0.net.0") == ("up1", 3) and split_level("up2.1.1.net.3") == ("up2", 2)
    for name in ("stage4.0.net.0", "up1.0.net.0", "up1.1.0.downsample.0", "stem.0", "stage4.1.downsample.0"):
        assert split_level(name) is None
    # one offset per accumulation group (64 // (3 ceil(cin / 16)) <= 1) from Cin 176 up: the split is exact only there
    assert [c for c in range(16, 400, 16) if one_offset_per_group(c)][0] == 176
