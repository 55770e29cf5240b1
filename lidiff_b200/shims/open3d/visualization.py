"""`draw_geometries` without a display (lidiff/vis_pcd.py:18): the point clouds are rendered on the GPU by lidiff_b200.render and
written as `<window_name>_<k>.png` into $LB2_O3D_RENDER_DIR (default: the working directory), k the first index whose file does
not exist yet; the path is printed.  The camera is open3d 0.17's default view of the clouds' bounding box unless lookat / up /
front / zoom are given.  All clouds share one image: they are drawn in their colours when every cloud has colours, else by
open3d's jet colour map of the height, and shaded with their normals when every cloud has normals."""
import os

import numpy as np

from .geometry import PointCloud

RENDER_DIR_ENV = "LB2_O3D_RENDER_DIR"


def _next_path(directory, window_name):
    k = 0
    while os.path.exists(os.path.join(directory, f"{window_name}_{k}.png")):
        k += 1
    return os.path.join(directory, f"{window_name}_{k}.png")


def draw_geometries(geometry_list, window_name="Open3D", width=1920, height=1080, left=50, top=50, point_show_normal=False,
                    mesh_show_wireframe=False, mesh_show_back_face=False, lookat=None, up=None, front=None, zoom=None):
    from lidiff_b200.render import Camera, render, write_png
    if point_show_normal:
        raise NotImplementedError("open3d shim: draw_geometries draws no normal lines (point_show_normal=True)")
    if mesh_show_wireframe or mesh_show_back_face:
        raise NotImplementedError("open3d shim: draw_geometries draws point clouds only (mesh_show_wireframe / mesh_show_back_face)")
    clouds = list(geometry_list)
    for g in clouds:
        if not isinstance(g, PointCloud):
            raise NotImplementedError(f"open3d shim: draw_geometries draws point clouds only, got {type(g).__name__}")
    pts = [np.asarray(g.points, dtype=np.float64).reshape(-1, 3) for g in clouds]
    allpts = np.concatenate(pts) if pts else np.zeros((0, 3))
    normals = np.concatenate([np.asarray(g.normals) for g in clouds]) if clouds and all(g.has_normals() for g in clouds) else None
    colors = (np.concatenate([np.asarray(g.colors) for g in clouds])
              if clouds and all(g.has_colors() for g in clouds) else None)
    cam = Camera.fit(allpts, lookat=lookat, front=front, up=up, zoom=zoom, width=width, height=height)
    rgb = render(allpts, cam, normals=normals, colors=colors)
    directory = os.environ.get(RENDER_DIR_ENV) or os.getcwd()
    path = write_png(_next_path(directory, window_name), rgb)
    print(f"draw_geometries: wrote {path}")
    return path
