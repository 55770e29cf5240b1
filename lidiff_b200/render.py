"""Point-cloud images on the GPU without a display — the view that the reference's `lidiff/vis_pcd.py` opens with
`o3d.visualization.draw_geometries`, written as an 8-bit RGB PNG instead of shown in a window:

  * `Camera.fit(points, ...)`: open3d 0.17's default `ViewControl` from memory (the bounding box of the finite points, lookat = its
    centre, front = (0, 0, 1), up = (0, 1, 0), zoom = 0.7, a 60 degree vertical field of view, distance = zoom max_extent / tan(fov / 2));
  * `render(points, camera, normals, colors, point_size, z_range)`: square points of `point_size` pixels into a depth-keyed z-buffer
    (lb2_render_splat), then one shading pass per pixel (lb2_render_shade): the points' colours, or open3d's jet colour map of the
    height over `z_range`, times a two-sided headlight of the normals.  Deterministic: the nearest point wins each pixel, ties go to
    the lower index.  Pixels match open3d's window only in layout, not in lighting (DESIGN.md §5);
  * `write_png(path, rgb)`: an 8-bit RGB PNG written with the standard library.

Points may be numpy arrays, torch tensors on any device, or open3d-shim PointClouds.  There is no CPU fallback."""
from __future__ import annotations

import ctypes
import dataclasses
import math
import os
import struct
import zlib

import numpy as np
import torch

from . import _lib
from .metrics import _points, _xyz

DEFAULT_FRONT = (0.0, 0.0, 1.0)
DEFAULT_UP = (0.0, 1.0, 0.0)
DEFAULT_ZOOM = 0.7
DEFAULT_FOV = 60.0
BACKGROUND = 255


def _vec3(v, what) -> tuple:
    a = np.asarray(v, dtype=np.float64).reshape(-1)
    if a.shape != (3,) or not np.isfinite(a).all():
        raise ValueError(f"camera {what} must be 3 finite numbers, got {v!r}")
    return tuple(float(x) for x in a)


def _size(v, what) -> int:
    if int(v) != v or int(v) <= 0:
        raise ValueError(f"{what} must be a positive integer, got {v!r}")
    return int(v)


def finite_bounds(points) -> tuple[np.ndarray, np.ndarray] | None:
    """(min, max) fp64 (3,) of the rows whose coordinates are all finite; None without such a row"""
    p = torch.as_tensor(_xyz(points)).to(torch.float64)
    p = p[torch.isfinite(p).all(1)]
    if p.shape[0] == 0:
        return None
    return p.min(0).values.cpu().numpy(), p.max(0).values.cpu().numpy()


@dataclasses.dataclass(frozen=True)
class Camera:
    """A pinhole camera at lookat + normalize(front) distance, looking at `lookat`; `fov` is the vertical field of view in degrees."""
    lookat: tuple
    front: tuple
    up: tuple
    distance: float
    width: int = 1920
    height: int = 1080
    fov: float = DEFAULT_FOV

    def __post_init__(self):
        for name in ("lookat", "front", "up"):
            object.__setattr__(self, name, _vec3(getattr(self, name), name))
        object.__setattr__(self, "width", _size(self.width, "image width"))
        object.__setattr__(self, "height", _size(self.height, "image height"))
        f, u = np.array(self.front), np.array(self.up)
        if not np.any(f):
            raise ValueError("camera front must not be the zero vector")
        if not np.any(u):
            raise ValueError("camera up must not be the zero vector")
        if not np.any(np.cross(u, f)):
            raise ValueError(f"camera up {self.up} is parallel to front {self.front}")
        if not (math.isfinite(self.distance) and self.distance > 0):
            raise ValueError(f"camera distance must be positive and finite, got {self.distance!r}")
        if not 0 < self.fov < 180:
            raise ValueError(f"field of view must be in (0, 180) degrees, got {self.fov!r}")

    @property
    def focal(self) -> float:
        """pixels per unit of x / depth: (height / 2) / tan(fov / 2)"""
        return (self.height / 2.0) / math.tan(math.radians(self.fov) / 2.0)

    @classmethod
    def fit(cls, points, lookat=None, front=None, up=None, zoom=None, width=1920, height=1080, fov=DEFAULT_FOV) -> "Camera":
        """open3d's default view of the finite points' bounding box; each given argument overrides its default (a cloud without a
        finite point is treated as the unit box at the origin, a single point as a box of extent 1)"""
        b = finite_bounds(points)
        lo, hi = b if b is not None else (np.zeros(3), np.ones(3))
        zoom = DEFAULT_ZOOM if zoom is None else float(zoom)
        if not (math.isfinite(zoom) and zoom > 0):
            raise ValueError(f"zoom must be positive and finite, got {zoom!r}")
        if not 0 < fov < 180:
            raise ValueError(f"field of view must be in (0, 180) degrees, got {fov!r}")
        extent = float((hi - lo).max())
        extent = extent if extent > 0 and math.isfinite(extent) else 1.0
        return cls(lookat=(lo + hi) / 2.0 if lookat is None else lookat, front=DEFAULT_FRONT if front is None else front,
                   up=DEFAULT_UP if up is None else up, distance=zoom * extent / math.tan(math.radians(fov) / 2.0),
                   width=width, height=height, fov=fov)

    def c_struct(self) -> _lib.RenderCamera:
        v3 = lambda v: (ctypes.c_double * 3)(*v)
        return _lib.RenderCamera(v3(self.lookat), v3(self.front), v3(self.up), float(self.distance), float(self.focal), self.width,
                                 self.height)


def _rows(x, n, what, device) -> torch.Tensor | None:
    if x is None:
        return None
    shape = tuple(x.shape) if isinstance(x, (np.ndarray, torch.Tensor)) else np.shape(np.asarray(x))
    if len(shape) != 2 or shape[1] != 3:
        raise ValueError(f"render: {what} must be an (n, 3) array, got shape {shape}")
    t = _points(x, device)
    if t.shape[0] != n:
        raise ValueError(f"render: {what} of shape {tuple(t.shape)} for {n} points")
    return t


def render(points, camera: Camera, normals=None, colors=None, point_size: float = 5.0, z_range=None, device="cuda") -> torch.Tensor:
    """(height, width, 3) uint8 device tensor of the cloud seen by `camera`: white background; each point a square of
    `point_size` pixels in its colour (fp64 (n, 3) in [0, 1]) or, without colours, open3d's jet of (z - z_lo) / (z_hi - z_lo)
    (z_range = (z_lo, z_hi), default the finite points' z range; heights outside it take the colour of its nearer end); with normals, times 0.25 + 0.75 |n . front|"""
    if not isinstance(camera, Camera):
        raise ValueError(f"render: camera must be a lidiff_b200.render.Camera, got {type(camera).__name__}")
    s = float(point_size)
    if not (s > 0 and s <= 4096):
        raise ValueError(f"render: point_size must be in (0, 4096], got {point_size!r}")
    h = _lib.get_handle(device)
    p = _points(points, h.device)
    if p.shape[1] != 3:
        raise ValueError(f"render: expected (n, 3) points, got shape {tuple(p.shape)}")
    n = p.shape[0]
    nrm, col = _rows(normals, n, "normals", h.device), _rows(colors, n, "colors", h.device)
    if z_range is None:
        b = finite_bounds(p)
        z_lo, z_hi = (float(b[0][2]), float(b[1][2])) if b is not None else (0.0, 0.0)
    else:
        z_lo, z_hi = (float(v) for v in z_range)
        if not (math.isfinite(z_lo) and math.isfinite(z_hi) and z_lo <= z_hi):
            raise ValueError(f"render: z_range must be two finite numbers, low <= high, got {z_range!r}")
    cam = camera.c_struct()
    rgb = torch.empty((camera.height, camera.width, 3), dtype=torch.uint8, device=h.device)
    if n == 0:
        rgb.fill_(BACKGROUND)
        return rgb
    keys = torch.full((camera.height * camera.width,), -1, dtype=torch.int64, device=h.device)
    h.render_splat(p, cam, s, keys)
    h.render_shade(keys, p, nrm, col, z_lo, z_hi, cam, rgb)
    return rgb


def _chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def encode_png(rgb) -> bytes:
    """an 8-bit RGB PNG (filter 0 on every row) of the (height, width, 3) uint8 image"""
    a = rgb.cpu().numpy() if isinstance(rgb, torch.Tensor) else np.asarray(rgb)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[0] == 0 or a.shape[1] == 0:
        raise ValueError(f"write_png: expected a non-empty (height, width, 3) uint8 image, got {a.dtype} {a.shape}")
    hgt, wid = a.shape[:2]
    raw = np.concatenate([np.zeros((hgt, 1), np.uint8), np.ascontiguousarray(a).reshape(hgt, 3 * wid)], axis=1).tobytes()
    return (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", wid, hgt, 8, 2, 0, 0, 0))
            + _chunk(b"IDAT", zlib.compress(raw, 6)) + _chunk(b"IEND", b""))


def write_png(path: str, rgb) -> str:
    """write the (height, width, 3) uint8 image (device or host) to `path` as an 8-bit RGB PNG; returns the path"""
    data = encode_png(rgb)
    d = os.path.dirname(os.path.abspath(path))
    os.makedirs(d, exist_ok=True)
    with open(path, "wb") as f:
        f.write(data)
    return path
