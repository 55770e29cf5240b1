"""open3d's uniform surface sampling of triangle meshes on the GPU, bit for bit — what the reference's metrics call to score a mesh
prediction (lidiff/utils/metrics.py:37, `geom.sample_points_uniformly(1000000)` in Metrics3D.convert_to_pcd).

    pts, key, pos = sample_points_uniformly(vertices, triangles, 1_000_000, key, pos)

restates open3d 0.17's TriangleMesh::SamplePointsUniformly under libstdc++ (include/lidiff_b200.h gives every formula and its
order): the triangle areas, their left-to-right sum S, the sequential cdf of area / S, n_t = round(cdf_t N) points on triangle t,
and for each point two `uniform_real_distribution<double>(0, 1)` draws of a `std::mt19937`, four 32-bit words, drawn on the device
by lb2_mt19937_words.  The stream is explicit: (key, pos) is numpy's legacy MT19937 state (624 words, position), and the call
returns the state after exactly 4 N words.  `std::mt19937(s)` is numpy's legacy seeding of s (`seed_state`).

Input the reference's program could not sample raises before any sampling launch or word is drawn: N <= 0, no triangles, a vertex
index outside [0, n_vertices), a NaN / inf vertex used by a triangle, and S == 0 (or not finite) raise ValueError; an allocation
whose last n_t is not N (impossible while n_triangles N < 2^51) raises RuntimeError.  There is no CPU fallback.
"""
from __future__ import annotations

import os
import threading

import numpy as np
import torch

from . import _lib
from .rng import MT_N, _words

_INFO = np.dtype([("surface_area", "<f8"), ("last_count", "<i8"), ("status", "<i4"), ("pad", "<i4")])    # lb2_mesh_info


def seed_state(seed: int) -> tuple[np.ndarray, int]:
    """(key, pos) of `std::mt19937(seed)`: the seed taken modulo 2^32, as libstdc++'s engine does (numpy's legacy seeding)"""
    _, key, pos, _, _ = np.random.RandomState(int(seed) % (1 << 32)).get_state(legacy=True)
    return np.asarray(key, np.uint32).copy(), int(pos)


def _mesh(vertices, triangles, device):
    """(fp64 (n, 3), int32 (m, 3)) contiguous device tensors; an index outside int32's range is outside [0, n) and raises here"""
    v = vertices.detach() if isinstance(vertices, torch.Tensor) else torch.as_tensor(np.asarray(vertices, dtype=np.float64))
    t = triangles.detach().cpu().numpy() if isinstance(triangles, torch.Tensor) else np.asarray(triangles)
    if v.dim() != 2 or v.shape[1] != 3 or t.ndim != 2 or t.shape[1] != 3:
        raise ValueError(f"expected (n, 3) vertices and (m, 3) triangles, got {tuple(v.shape)} and {t.shape}")
    if t.dtype.kind not in "iu":
        raise ValueError(f"triangles must hold integer vertex indices, got {t.dtype}")
    if t.shape[0] == 0:
        raise ValueError("the mesh has no triangles")
    if t.dtype != np.int32:
        if int(t.min()) < 0 or int(t.max()) >= min(v.shape[0], 1 << 31):
            raise ValueError(f"a vertex index lies outside [0, {v.shape[0]})")
        t = t.astype(np.int32)
    return (v.to(device=device, dtype=torch.float64).contiguous(),
            torch.from_numpy(np.ascontiguousarray(t)).to(device=device))


def _prepare(h, v, t, n):
    """the areas, S and the n_t (in scratch) on the device, and the one status read: (scratch, S); raises on bad input"""
    area = torch.empty(t.shape[0], dtype=torch.float64, device=h.device)
    info = torch.empty(_INFO.itemsize, dtype=torch.uint8, device=h.device)
    scratch = h.mesh_sample_scratch(t.shape[0])
    h.mesh_sample_prepare(v, t, n, area, info, scratch)
    rec = np.frombuffer(info.cpu().numpy().tobytes(), _INFO)[0]
    status, s = int(rec["status"]), float(rec["surface_area"])
    if status & _lib.MESH_BAD_INDEX:
        raise ValueError(f"a vertex index lies outside [0, {v.shape[0]})")
    if status & _lib.MESH_NON_FINITE:
        raise ValueError("a triangle uses a vertex with a NaN or infinite coordinate")
    if status & _lib.MESH_BAD_AREA:
        raise ValueError(f"the mesh's surface area is {s}: nothing to sample")
    if status & _lib.MESH_BAD_COUNT:
        raise RuntimeError(f"the triangles hold {int(rec['last_count'])} of the {n} points (n_triangles x n_points too large)")
    return scratch, s


def surface_area(vertices, triangles, device="cuda") -> float:
    """S = the sum of the triangle areas, left to right (TriangleMesh::GetSurfaceArea); raises as sample_points_uniformly does"""
    h = _lib.get_handle(device)
    v, t = _mesh(vertices, triangles, h.device)
    return _prepare(h, v, t, 1)[1]


def sample_points_uniformly(vertices, triangles, number_of_points: int, key, pos: int, device="cuda"):
    """(points fp64 (N, 3) on `device`, key after, pos after) of open3d's SamplePointsUniformly(N) on the mesh (vertices (n, 3),
    integer triangles (m, 3)) with the std::mt19937 at numpy state (key, pos); the state afterwards is 4 N words further"""
    n = int(number_of_points)
    if n <= 0:
        raise ValueError(f"number_of_points must be > 0, got {n}")
    key = np.array(key, np.uint32)                                   # a copy: the word generator updates its state in place
    if key.shape != (MT_N,) or not 0 <= int(pos) <= MT_N:
        raise ValueError(f"an MT19937 state is {MT_N} words and a position in [0, {MT_N}]")
    h = _lib.get_handle(device)
    v, t = _mesh(vertices, triangles, h.device)
    scratch, _ = _prepare(h, v, t, n)
    words, state, pos2 = _words(h, key, int(pos), 4 * n)
    out = torch.empty((n, 3), dtype=torch.float64, device=h.device)
    h.mesh_sample_points(v, t, scratch, words, n, out)
    return out, state.cpu().numpy().view(np.uint32).copy(), int(pos2)


class GlobalStream:
    """the process-wide std::mt19937 of open3d's utility::random: seeded from 32 bits of OS entropy on first use unless `seed` was
    called (open3d seeds from std::random_device, so an unseeded run is not reproducible either)"""

    def __init__(self):
        self._lock = threading.Lock()
        self._state = None

    def seed(self, seed: int):
        with self._lock:
            self._state = seed_state(seed)

    def _current(self):
        if self._state is None:
            self._state = seed_state(int.from_bytes(os.urandom(4), "little"))
        return self._state

    def state(self) -> tuple[np.ndarray, int]:
        """(key, pos) now"""
        with self._lock:
            key, pos = self._current()
            return key.copy(), pos

    def sample_points_uniformly(self, vertices, triangles, number_of_points, device="cuda") -> torch.Tensor:
        """sample_points_uniformly on this stream, which advances by 4 N words (not at all when the call raises)"""
        with self._lock:
            pts, key, pos = sample_points_uniformly(vertices, triangles, number_of_points, *self._current(), device=device)
            self._state = (key, pos)
        return pts


STREAM = GlobalStream()
