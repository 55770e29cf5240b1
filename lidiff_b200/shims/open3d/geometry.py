import numpy as np

from .utility import Vector3dVector, Vector3iVector


class KDTreeSearchParamKNN:
    def __init__(self, knn=30):
        self.knn = int(knn)


class KDTreeSearchParamHybrid:
    def __init__(self, radius, max_nn):
        self.radius, self.max_nn = float(radius), int(max_nn)


class Geometry:
    """base class (lidiff/utils/metrics.py tests isinstance(geom, o3d.geometry.Geometry))"""


class GeometryType:
    class _T:
        def __init__(self, v):
            self.value = v
    Unspecified, PointCloud, VoxelGrid = _T(0), _T(1), _T(2)
    TriangleMesh = _T(6)


def _knn(query, ref, k):
    """exact k nearest neighbours of `query` (m,3) among `ref` (n,3), torch tensors on one device -> (dist (m,k), idx (m,k)).
    Bucketed search: queries are sorted into cells of the k-th-neighbour scale; a chunk of consecutive queries searches only the
    reference points inside its bounding box grown by the current margin and is redone with a larger margin if some k-th distance
    exceeds it (so every true neighbour lies inside the searched box).  O(m * local density) instead of O(m * n)."""
    import torch
    m, n = query.shape[0], ref.shape[0]
    k = min(k, n)
    lo, hi = torch.minimum(query.min(0).values, ref.min(0).values), torch.maximum(query.max(0).values, ref.max(0).values)
    vol = float(torch.clamp(hi - lo, min=1e-3).prod())
    cell = max((vol * max(k, 8) / max(n, 1)) ** (1.0 / 3.0), 1e-3)           # a cell holds ~k reference points at the mean density
    ijk = torch.floor((query - lo) / cell).long()
    dims = ijk.max(0).values + 1
    order = torch.argsort((ijk[:, 2] * dims[1] + ijk[:, 1]) * dims[0] + ijk[:, 0])
    qs = query[order]
    dist = torch.empty((m, k), dtype=query.dtype, device=query.device)
    idx = torch.empty((m, k), dtype=torch.long, device=query.device)
    all_ids = torch.arange(n, device=query.device)
    chunk = 4096
    for a in range(0, m, chunk):
        q = qs[a:a + chunk]
        qlo, qhi = q.min(0).values, q.max(0).values
        margin = 2.0 * cell
        while True:
            sel = ((ref >= qlo - margin) & (ref <= qhi + margin)).all(1)
            cand = ref[sel]
            whole = cand.shape[0] == n
            if cand.shape[0] >= k:
                d, j = torch.cdist(q, cand).topk(k, dim=1, largest=False)
                if whole or float(d[:, -1].max()) <= margin:
                    break
            margin *= 2.0
        dist[order[a:a + chunk]] = d
        idx[order[a:a + chunk]] = all_ids[sel][j]
    return dist, idx


class VoxelGrid(Geometry):
    """`VoxelGrid.create_from_point_cloud(pcd, voxel_size)` + `check_if_included(points)` (lidiff/utils/collations.py:44-50,
    eval_path.py:95-100): open3d puts the grid origin at the cloud's minimum bound minus half a voxel and marks the voxels that
    contain at least one point; a query is included when its voxel floor((p - origin) / voxel_size) is marked."""

    def __init__(self):
        self.voxel_size, self.origin, self._keys = 0.0, np.zeros(3), np.zeros((0, 3), np.int64)

    @staticmethod
    def create_from_point_cloud(input, voxel_size):
        g = VoxelGrid()
        pts = np.asarray(input.points, dtype=np.float64)
        g.voxel_size = float(voxel_size)
        g.origin = pts.min(0) - 0.5 * g.voxel_size if len(pts) else np.zeros(3)
        g._keys = np.unique(np.floor((pts - g.origin) / g.voxel_size).astype(np.int64), axis=0) if len(pts) else g._keys
        return g

    def get_geometry_type(self):
        return GeometryType.VoxelGrid

    def get_voxels(self):
        return [tuple(k) for k in self._keys]

    def check_if_included(self, queries):
        q = np.floor((np.asarray(queries, dtype=np.float64) - self.origin) / self.voxel_size).astype(np.int64)
        if len(self._keys) == 0:
            return [False] * len(q)
        span = np.maximum(self._keys.max(0), q.max(0)) - np.minimum(self._keys.min(0), q.min(0)) + 1
        base = np.minimum(self._keys.min(0), q.min(0))
        enc = lambda v: ((v[:, 0] - base[0]) * span[1] + (v[:, 1] - base[1])) * span[2] + (v[:, 2] - base[2])
        return np.isin(enc(q), enc(self._keys)).tolist()


class PointCloud(Geometry):
    def __init__(self, points=None):
        self._points = Vector3dVector(points if points is not None else ())
        self._normals = Vector3dVector(())
        self._colors = Vector3dVector(())

    points = property(lambda s: s._points, lambda s, v: setattr(s, "_points", Vector3dVector(v)))
    normals = property(lambda s: s._normals, lambda s, v: setattr(s, "_normals", Vector3dVector(v)))
    colors = property(lambda s: s._colors, lambda s, v: setattr(s, "_colors", Vector3dVector(v)))

    def has_points(self):
        return len(self._points) > 0

    def has_normals(self):
        return len(self._normals) == len(self._points) > 0

    def has_colors(self):
        return len(self._colors) == len(self._points) > 0

    def paint_uniform_color(self, color):
        """every point gets the RGB `color` (3 values in [0, 1])"""
        c = np.asarray(color, dtype=np.float64).reshape(-1)
        if c.shape != (3,):
            raise ValueError(f"paint_uniform_color: expected 3 values, got {color!r}")
        self._colors = Vector3dVector(np.broadcast_to(c, (len(self._points), 3)).copy())
        return self

    def __repr__(self):
        return f"PointCloud with {len(self._points)} points."

    def farthest_point_down_sample(self, num_samples):
        """open3d 0.17 semantics: start at index 0, repeatedly add the point farthest from the selected set (first index on
        ties); like open3d's SelectByIndex the result lists the selected points in ORIGINAL index order.  GPU only
        (lb2_farthest_point_sample); no CPU fallback."""
        import torch
        from lidiff_b200.preprocess import farthest_point_sample
        if not torch.cuda.is_available():
            raise RuntimeError("open3d shim: farthest_point_down_sample needs the lidiff_b200 CUDA library and a GPU")
        n = int(num_samples)
        if n <= 0 or n > len(self._points):
            raise RuntimeError("Illegal number of samples")
        sel = farthest_point_sample(torch.as_tensor(np.asarray(self._points), device="cuda"), n)
        out = PointCloud(np.asarray(self._points)[sel.cpu().numpy()])
        if self.has_normals():
            out.normals = np.asarray(self._normals)[sel.cpu().numpy()]
        return out

    def compute_point_cloud_distance(self, target):
        """for every point of this cloud the Euclidean distance to its nearest point of `target` (open3d: KDTreeFlann 1-NN in
        double precision) — what lidiff/utils/metrics.py builds RMSE / Chamfer distance / precision-recall on.  On a GPU: the exact
        fp64 tree search of the lidiff_b200 CUDA library (lidiff_b200.metrics.nn_distance)."""
        import torch
        if torch.cuda.is_available():
            from lidiff_b200.metrics import nn_distance
            if len(self._points) == 0 or len(target._points) == 0:
                return np.zeros(len(self._points))
            return nn_distance(np.asarray(self._points), np.asarray(target._points)).cpu().numpy()
        dev = "cpu"
        q64 = torch.as_tensor(np.asarray(self._points), dtype=torch.float64, device=dev)
        r64 = torch.as_tensor(np.asarray(target._points), dtype=torch.float64, device=dev)
        if q64.shape[0] == 0 or r64.shape[0] == 0:
            return np.zeros(q64.shape[0])
        _, idx = _knn(q64.float(), r64.float(), 1)
        # the neighbour found in fp32 can differ from the fp64 one only between candidates equidistant to 1e-7: re-evaluate in fp64
        return (q64 - r64[idx[:, 0]]).norm(dim=1).cpu().numpy()

    def get_geometry_type(self):
        return GeometryType.PointCloud

    def get_min_bound(self):
        return np.asarray(self._points).min(0)

    def get_max_bound(self):
        return np.asarray(self._points).max(0)

    def estimate_normals(self, search_param=None, fast_normal_computation=True):
        """PCA normal of the k nearest neighbours (k = `knn`, else `max_nn`, else 30 as open3d's default KNN search; the radius of
        KDTreeSearchParamHybrid is ignored), sign left unoriented.  On a GPU: open3d's cumulant covariance and FastEigen3x3 over an
        exact (d², index)-ordered k-NN (lidiff_b200.normals.estimate_normals); that kernel takes k <= 32, so a larger knn / max_nn
        raises ValueError there rather than running another implementation.  Without a GPU: an exact bucketed k-NN search (`_knn`)
        and the eigenvector of torch's eigh, any k."""
        import torch
        k = getattr(search_param, "knn", None) or getattr(search_param, "max_nn", None) or 30
        if torch.cuda.is_available():
            from lidiff_b200.normals import estimate_normals
            pts = np.asarray(self._points)
            self._normals = Vector3dVector(estimate_normals(pts, knn=k).cpu().numpy() if len(pts) else np.zeros((0, 3)))
            return True
        dev = "cpu"
        p = torch.as_tensor(np.asarray(self._points), dtype=torch.float32, device=dev)
        n = p.shape[0]
        k = min(k, n)
        out = torch.zeros((n, 3), dtype=torch.float32, device=dev)
        if n >= 3:
            _, idx = _knn(p, p, k)
            for a in range(0, n, 65536):
                nb = p[idx[a:a + 65536]]                                              # (c, k, 3)
                c = nb - nb.mean(1, keepdim=True)
                cov = c.transpose(1, 2) @ c
                out[a:a + 65536] = torch.linalg.eigh(cov.double())[1][:, :, 0].float()   # eigenvector of the smallest eigenvalue
        self._normals = Vector3dVector(out.cpu().numpy())
        return True


class TriangleMesh(Geometry):
    """vertices (Vector3dVector) and triangles (Vector3iVector) — what lidiff/utils/metrics.py's Metrics3D reads from a mesh
    prediction.  `sample_points_uniformly` is open3d 0.17's, bit for bit, on the GPU (lidiff_b200.mesh) and draws from the global
    stream of `utility.random`.  Vertex normals and colours are not kept and not carried into the sampled cloud: the metrics never
    read them.  No CPU fallback."""

    def __init__(self, vertices=None, triangles=None):
        self._vertices = Vector3dVector(vertices if vertices is not None else ())
        self._triangles = Vector3iVector(triangles if triangles is not None else ())

    vertices = property(lambda s: s._vertices, lambda s, v: setattr(s, "_vertices", Vector3dVector(v)))
    triangles = property(lambda s: s._triangles, lambda s, v: setattr(s, "_triangles", Vector3iVector(v)))

    def __repr__(self):
        return f"TriangleMesh with {len(self._vertices)} points and {len(self._triangles)} triangles."

    def has_vertices(self):
        return len(self._vertices) > 0

    def has_triangles(self):
        return len(self._vertices) > 0 and len(self._triangles) > 0

    def get_geometry_type(self):
        return GeometryType.TriangleMesh

    def get_surface_area(self):
        """the sum of the triangle areas, left to right, as open3d adds them (lidiff_b200.mesh.surface_area)"""
        from lidiff_b200.mesh import surface_area
        return surface_area(np.asarray(self._vertices), np.asarray(self._triangles))

    def sample_points_uniformly(self, number_of_points=100, use_triangle_normal=False):
        """a PointCloud of `number_of_points` points drawn uniformly from the surface (open3d's SamplePointsUniformly); the global
        stream of utility.random advances by 4 number_of_points words.  Raises ValueError for number_of_points <= 0, a mesh without
        triangles, a vertex index out of range, a NaN / inf vertex of a triangle or a zero surface area."""
        if use_triangle_normal:
            raise NotImplementedError("open3d shim: sample_points_uniformly carries no normals (use_triangle_normal=True)")
        from lidiff_b200.mesh import STREAM
        pts = STREAM.sample_points_uniformly(np.asarray(self._vertices), np.asarray(self._triangles), number_of_points)
        return PointCloud(pts.cpu().numpy())
