"""Minimal `open3d` for the reference's inference script (SURVEY.md 8f-1/8f-2; diff_completion_pipeline.py:97-99,175,204-212):
`geometry.PointCloud` (points / normals, `farthest_point_down_sample`, `estimate_normals`), `utility.Vector3dVector`,
`io.read_point_cloud` / `io.write_point_cloud` for PLY.  Farthest point sampling runs on the GPU through
lb2_farthest_point_sample (same first-index start and first-argmax tie rule as open3d 0.17).  For lidiff/vis_pcd.py:
`visualization.draw_geometries` renders point clouds on the GPU to PNG files instead of opening a window (lidiff_b200.render), and
`PointCloud.paint_uniform_color` sets every point's colour.  For mesh predictions (lidiff/utils/metrics.py:31-52):
`geometry.TriangleMesh` whose `sample_points_uniformly` is open3d's on the GPU (lidiff_b200.mesh), `utility.Vector3iVector`,
`utility.random.seed` and `io.read_triangle_mesh` for PLY."""
from . import geometry, io, utility, visualization  # noqa: F401

__version__ = "0.17.0+lidiff_b200.shim"
