"""numpy restatement of open3d 0.17's TriangleMesh::SamplePointsUniformly under libstdc++ (the contract of csrc/mesh.cu in
include/lidiff_b200.h), the oracle of the mesh tests:

  * areas: 0.5 |x × y|, x = p0 - p1, y = p0 - p2, |c| = sqrt((c0² + c1²) + c2²), every operation rounded on its own;
  * S = area_0 + area_1 + ... and cdf_t = area_t / S + cdf_{t-1}, both left to right (np.add.accumulate is sequential);
  * n_t = round(cdf_t N), half away from zero; point i lies on the first t with n_t > i;
  * r = RN(w_lo + w_hi 2^32) 2^-64 (nextafter(1, 0) when r >= 1) for r1, then r2, from words 4i .. 4i+3 of the std::mt19937;
  * s = sqrt(r1), a = 1 - s, b = s (1 - r2), c = s r2, p = (a v0 + b v1) + c v2.

numpy evaluates each elementwise operation on its own (no FMA contraction), which is what the kernels do with __d*_rn.
`sample_loop` is a literal per-point transcription of open3d's loop, used to pin the vectorised `sample` on small meshes."""
import math

import numpy as np

import rng_reference as R

NEXT_BELOW_ONE = np.nextafter(1.0, 0.0)


def areas(verts, tris) -> np.ndarray:
    v = np.asarray(verts, np.float64)
    t = np.asarray(tris, np.int64)
    p0, p1, p2 = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    with np.errstate(over="ignore", invalid="ignore"):             # huge or non-finite coordinates give inf / NaN areas
        x, y = p0 - p1, p0 - p2
        c0 = x[:, 1] * y[:, 2] - x[:, 2] * y[:, 1]
        c1 = x[:, 2] * y[:, 0] - x[:, 0] * y[:, 2]
        c2 = x[:, 0] * y[:, 1] - x[:, 1] * y[:, 0]
        return 0.5 * np.sqrt((c0 * c0 + c1 * c1) + c2 * c2)


def surface_area(a) -> float:
    return float(np.add.accumulate(np.asarray(a, np.float64))[-1])


def round_half_away(x) -> np.ndarray:
    """std::round for x >= 0: the fraction x - floor(x) is exact"""
    f = np.floor(x)
    return np.where(x - f >= 0.5, f + 1.0, f)


def counts(a, n) -> np.ndarray:
    """n_t (int64) of the areas `a` for N = n"""
    a = np.asarray(a, np.float64)
    cdf = np.add.accumulate(a / surface_area(a))
    return round_half_away(cdf * float(n)).astype(np.int64)


def canonical(lo, hi) -> np.ndarray:
    r = (np.asarray(lo, np.uint32).astype(np.float64) + np.asarray(hi, np.uint32).astype(np.float64) * 2.0 ** 32) * 2.0 ** -64
    return np.where(r >= 1.0, NEXT_BELOW_ONE, r)


def sample(verts, tris, n, words) -> np.ndarray:
    """(n, 3) fp64 points from the 4n uint32 `words`"""
    v = np.asarray(verts, np.float64)
    t = np.asarray(tris, np.int64)
    w = np.asarray(words, np.uint32)[: 4 * n].reshape(n, 4)
    tri = np.searchsorted(counts(areas(v, t), n), np.arange(n), side="right")
    r1, r2 = canonical(w[:, 0], w[:, 1]), canonical(w[:, 2], w[:, 3])
    s = np.sqrt(r1)
    a, b, c = 1.0 - s, s * (1.0 - r2), s * r2
    p0, p1, p2 = v[t[tri, 0]], v[t[tri, 1]], v[t[tri, 2]]
    return (a[:, None] * p0 + b[:, None] * p1) + c[:, None] * p2


def sample_stream(verts, tris, n, key, pos):
    """(points, key after, pos after) with the words of the MT19937 state (key, pos)"""
    words, key2, pos2 = R.mt_words(key, pos, 4 * n)
    return sample(verts, tris, n, words), key2, pos2


def sample_loop(verts, tris, n, words) -> np.ndarray:
    """open3d's SamplePointsUniformlyImpl, one point at a time in Python floats (IEEE doubles, no FMA)"""
    v = [tuple(float(c) for c in row) for row in np.asarray(verts, np.float64)]
    t = [tuple(int(i) for i in row) for row in np.asarray(tris)]
    area = []
    for i0, i1, i2 in t:
        x = [v[i0][k] - v[i1][k] for k in range(3)]
        y = [v[i0][k] - v[i2][k] for k in range(3)]
        c = (x[1] * y[2] - x[2] * y[1], x[2] * y[0] - x[0] * y[2], x[0] * y[1] - x[1] * y[0])
        area.append(0.5 * math.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]))
    s = 0.0
    for a in area:
        s += a
    cdf = [area[0] / s]
    for a in area[1:]:
        cdf.append(a / s + cdf[-1])
    it = iter(int(x) for x in np.asarray(words, np.uint32)[: 4 * n])

    def uniform():
        lo, hi = next(it), next(it)
        r = (float(lo) + float(hi) * 2.0 ** 32) * 2.0 ** -64
        return r if r < 1.0 else float(NEXT_BELOW_ONE)

    out, i = np.zeros((n, 3)), 0
    for ti, (i0, i1, i2) in enumerate(t):
        x = cdf[ti] * n
        nt = math.floor(x) + (1 if x - math.floor(x) >= 0.5 else 0)              # std::round
        while i < nt:
            r1 = uniform()
            r2 = uniform()
            a, b, c = 1 - math.sqrt(r1), math.sqrt(r1) * (1 - r2), math.sqrt(r1) * r2
            out[i] = [(a * v[i0][k] + b * v[i1][k]) + c * v[i2][k] for k in range(3)]
            i += 1
    return out


def height_field(side: int, seed: int = 0, offset: float = 0.0):
    """(vertices, triangles) of a side x side-vertex height field on a 0.1 m grid, z = a smooth surface plus seeded noise, shifted
    by `offset` in x and y: 2 (side - 1)^2 triangles"""
    g = np.random.default_rng(seed)
    ij = np.stack(np.meshgrid(np.arange(side), np.arange(side), indexing="ij"), -1).reshape(-1, 2).astype(np.float64)
    z = np.sin(ij[:, 0] * 0.05) * np.cos(ij[:, 1] * 0.03) + g.normal(0.0, 0.02, ij.shape[0])
    verts = np.stack([ij[:, 0] * 0.1 + offset, ij[:, 1] * 0.1 + offset, z], 1)
    q = (np.arange(side - 1)[:, None] * side + np.arange(side - 1)[None, :]).reshape(-1)
    tris = np.concatenate([np.stack([q, q + side, q + 1], 1), np.stack([q + 1, q + side, q + side + 1], 1)]).astype(np.int32)
    return verts, tris
