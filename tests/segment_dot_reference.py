"""TEST INFRASTRUCTURE: lb2_segment_dot's documented summation order restated in numpy (include/lidiff_b200.h), the yardstick of the
GPU test, and its fp32 error bound against an exact sum.

Order, per channel: chunk k is the positions [k R, (k + 1) R) of the row order; a piece is a non-empty intersection of a segment
with a chunk; a piece's sum is ((+0 + p_b) + p_b+1) + ... over its products p_i = RN(a_i b_i) in ascending position; a segment with one
piece is that sum, one with several is ((+0 + piece_0) + piece_1) + ... in ascending chunk order, one without rows is +0."""
import numpy as np

R = 128          # LB2_SEGMENT_DOT_R


def _fold(rows):
    """((+0 + r_0) + r_1) + ... with one fp32 rounding per add (np.add.accumulate is that recurrence; np.sum adds pairwise)"""
    return np.add.accumulate(np.concatenate([np.zeros((1, rows.shape[1]), np.float32), rows]), axis=0)[-1]


def pieces_of(offsets):
    """per segment, the list of (begin, end) positions of its pieces"""
    out = []
    for s in range(len(offsets) - 1):
        b, e = int(offsets[s]), int(offsets[s + 1])
        cuts = [b] + list(range((b // R + 1) * R, e, R)) + [e] if e > b else []
        out.append(list(zip(cuts[:-1], cuts[1:])))
    return out


def emulate(a, b, order, offsets):
    """numpy fp32 (nseg, c): lb2_segment_dot(a, b, order, offsets) bit for bit; b None: the plain sum of a's rows"""
    a = np.asarray(a, np.float32)
    rows = np.arange(a.shape[0]) if order is None else np.asarray(order)
    out = np.zeros((len(offsets) - 1, a.shape[1]), np.float32)
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        p = a[rows] if b is None else a[rows] * np.asarray(b, np.float32)[rows]
        for s, pieces in enumerate(pieces_of(offsets)):
            sums = [_fold(p[pb:pe]) for pb, pe in pieces]
            if len(sums) == 1:
                out[s] = sums[0]
            elif sums:
                out[s] = _fold(np.stack(sums))
    return out


def exact_and_bound(a, b, order, offsets):
    """(fp64 sums, element-wise bound on |lb2_segment_dot - fp64|): with u = 2^-24, every product is within u |a b| of exact (plus
    half the smallest subnormal), and a product goes through at most min(L, R) adds inside its piece and n_pieces adds of the piece
    sums, each within u of its result: |err| <= ((1 + u)^(1 + min(L, R) + n_pieces) - 1) S1 + L 2^-150, S1 = sum |a b|"""
    a64 = np.asarray(a, np.float64)
    rows = np.arange(a64.shape[0]) if order is None else np.asarray(order)
    p = a64[rows] if b is None else a64[rows] * np.asarray(b, np.float64)[rows]
    nseg = len(offsets) - 1
    ref, bound = np.zeros((nseg, a64.shape[1])), np.zeros((nseg, a64.shape[1]))
    u = 2.0 ** -24
    for s, pieces in enumerate(pieces_of(offsets)):
        if not pieces:
            continue
        lo, hi = pieces[0][0], pieces[-1][1]
        ref[s] = p[lo:hi].sum(0)
        n_ops = 1 + min(hi - lo, R) + len(pieces)
        bound[s] = ((1 + u) ** n_ops - 1) * np.abs(p[lo:hi]).sum(0) + (hi - lo) * 2.0 ** -150
    return ref, bound
