import numpy as np


class Vector3dVector(np.ndarray):
    """(n, 3) float64 array; `np.array(v)` / `np.asarray(v)` give the points back as open3d's does"""

    def __new__(cls, data=()):
        a = np.asarray(data, dtype=np.float64)
        if a.size == 0:
            a = a.reshape(0, 3)
        if a.ndim != 2 or a.shape[1] != 3:
            raise RuntimeError(f"Vector3dVector expects shape (n, 3), got {a.shape}")
        return np.ascontiguousarray(a).view(cls)


class Vector3iVector(np.ndarray):
    """(n, 3) int32 array (triangle vertex indices)"""

    def __new__(cls, data=()):
        a = np.asarray(data)
        if a.size == 0:
            a = np.zeros((0, 3), np.int32)
        if a.ndim != 2 or a.shape[1] != 3:
            raise RuntimeError(f"Vector3iVector expects shape (n, 3), got {a.shape}")
        if a.dtype.kind not in "iu" or (a.size and (a.min() < -(1 << 31) or a.max() >= 1 << 31)):
            raise RuntimeError(f"Vector3iVector expects 32-bit integers, got {a.dtype}")
        return np.ascontiguousarray(a, dtype=np.int32).view(cls)


class random:  # noqa: N801  (open3d.utility.random is a module)
    """open3d.utility.random: the global std::mt19937 that TriangleMesh.sample_points_uniformly draws from (lidiff_b200.mesh.STREAM)"""

    @staticmethod
    def seed(seed: int):
        """std::mt19937(seed); seed is a C int, as in open3d"""
        s = int(seed)
        if not -(1 << 31) <= s < 1 << 31:
            raise TypeError(f"seed(): expected a 32-bit int, got {seed!r}")
        from lidiff_b200.mesh import STREAM
        STREAM.seed(s)
