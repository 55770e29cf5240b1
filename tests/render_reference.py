"""TEST INFRASTRUCTURE: a numpy restatement of lb2_render_splat and lb2_render_shade (include/lidiff_b200.h) in the header's
operation order: the fp64 camera basis and projection (every operation rounded on its own; numpy never contracts to FMA), the
footprint, the (float depth bits, index) minimum per pixel, then open3d's jet, the fp32 headlight and the byte rounding.  The GPU
tests compare the device's keys and bytes with it bit for bit; the host tests check it against closed forms."""
import math

import numpy as np

EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _normalize(a):
    l = math.sqrt(_dot(a, a))
    return (a[0] / l, a[1] / l, a[2] / l)


def basis(cam):
    """(F, right, up', eye) of a lidiff_b200.render.Camera, as Python floats (IEEE fp64, correctly rounded sqrt and division)"""
    f = _normalize(cam.front)
    r = _normalize(_cross(cam.up, f))
    u = _normalize(_cross(f, r))
    eye = tuple(cam.lookat[k] + f[k] * cam.distance for k in range(3))
    return f, r, u, eye


def project(pts, cam):
    """(depth, u, v, ok) fp64 (n,) each; ok = the point is finite, beyond the near rule and has a non-NaN u and v"""
    f, r, up, eye = basis(cam)
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        d = [p[:, k] - eye[k] for k in range(3)]
        depth = -_dot(d, f)
        u = 0.5 * cam.width + (cam.focal * _dot(d, r)) / depth
        v = 0.5 * cam.height - (cam.focal * _dot(d, up)) / depth
        ok = np.isfinite(p).all(1) & (depth > 1e-3 * cam.distance) & ~np.isnan(u) & ~np.isnan(v)
    return depth, u, v, ok


def span(centre, half, size):
    """[lo, hi) = the pixels c in [0, size) with centre - half <= c + 0.5 < centre + half (the header's clamped form)"""
    with np.errstate(invalid="ignore"):
        a = np.clip(np.asarray(centre, np.float64) - half, -1.0, size + 1.0)
        b = np.clip(np.asarray(centre, np.float64) + half, -1.0, size + 1.0)
        lo = np.maximum(np.ceil(a - 0.5), 0).astype(np.int64)
        hi = np.minimum(np.ceil(b - 0.5), size).astype(np.int64)
    return lo, hi


def splat(pts, cam, point_size, keys=None):
    """uint64 (height width,) z-buffer keys: per pixel min over covering points of (float32(depth) bits << 32) | index"""
    depth, u, v, ok = project(pts, cam)
    keys = np.full(cam.height * cam.width, EMPTY, np.uint64) if keys is None else keys
    idx = np.nonzero(ok)[0]
    if idx.shape[0] == 0:
        return keys
    half = 0.5 * float(point_size)
    i0, i1 = span(u[idx], half, cam.width)
    j0, j1 = span(v[idx], half, cam.height)
    with np.errstate(over="ignore"):                          # a depth beyond the fp32 range keys as +inf, as on the device
        key = (depth[idx].astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | idx.astype(np.uint64)
    reach = int(math.ceil(2 * half)) + 2
    for dj in range(reach):
        rj = j0 + dj
        mj = rj < j1
        if not mj.any():
            break
        for di in range(reach):
            ci = i0 + di
            m = mj & (ci < i1)
            if not m.any():
                if not (ci < i1).any():
                    break
                continue
            np.minimum.at(keys, rj[m] * cam.width + ci[m], key[m])
    return keys


def jet(t):
    """open3d's ColorMapJet of fp64 t: (JetBase(2t - 1.5), JetBase(2t - 1.0), JetBase(2t - 0.5)) in the header's operations"""
    t2 = np.asarray(t, np.float64) * 2.0

    def base(x):
        return np.where(x <= -0.75, 0.0, np.where(x <= -0.25, ((x - -0.75) / 0.5) * 1.0 + 0.0,
                        np.where(x <= 0.25, 1.0, np.where(x <= 0.75, ((x - 0.25) / 0.5) * -1.0 + 1.0, 0.0))))
    return np.stack([base(t2 - 1.5), base(t2 - 1.0), base(t2 - 0.5)], -1)


def shade(keys, pts, cam, normals=None, colors=None, z_lo=0.0, z_hi=0.0):
    """uint8 (height, width, 3) image of the keys"""
    rgb = np.full((cam.height * cam.width, 3), 255, np.uint8)
    hit = keys != EMPTY
    i = (keys[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    if colors is not None:
        c = np.asarray(colors, np.float64)[i].astype(np.float32)
    else:
        z = p[i, 2]
        t = np.zeros_like(z) if z_hi == z_lo else np.clip((z - z_lo) / (z_hi - z_lo), 0.0, 1.0)
        c = jet(t).astype(np.float32)
    k = np.ones(i.shape[0], np.float32)
    if normals is not None:
        f = basis(cam)[0]
        nv = np.asarray(normals, np.float64)[i]
        with np.errstate(invalid="ignore", over="ignore"):
            dot = _dot([nv[:, 0], nv[:, 1], nv[:, 2]], f).astype(np.float32)
            fin = np.isfinite(dot)
            k[fin] = np.float32(0.25) + np.float32(0.75) * np.abs(dot[fin])
    with np.errstate(invalid="ignore"):
        c = c * k[:, None]
        c = np.where(~(c > 0), np.float32(0), np.where(c > 1, np.float32(1), c)).astype(np.float32)
    rgb[hit] = np.rint(np.float32(255) * c).astype(np.uint8)
    return rgb.reshape(cam.height, cam.width, 3)


def render(pts, cam, normals=None, colors=None, point_size=5.0, z_range=None):
    """(keys, rgb) as lidiff_b200.render.render computes them"""
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    if z_range is None:
        fin = p[np.isfinite(p).all(1)]
        z_range = (float(fin[:, 2].min()), float(fin[:, 2].max())) if fin.shape[0] else (0.0, 0.0)
    keys = splat(p, cam, point_size)
    return keys, shade(keys, p, cam, normals, colors, *z_range)
