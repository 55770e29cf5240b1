"""Point-cloud views as PNG images — the counterpart of the reference's `python3 lidiff/vis_pcd.py -p cloud.ply -r 50`,
which opens an open3d window; this renders the same view on the GPU (lidiff_b200.render) and
writes it to a file, so a completion can be looked at on a machine without a display.

Like the reference: the points with |p| < radius and -2.5 < z < 3 are kept (radius > 0; radius <= 0 keeps every point), their
normals are estimated with open3d's 30-nearest-neighbour PCA (lidiff_b200.normals), and the cloud is drawn from open3d's default
camera with jet colours by height.  `-p` may also be a directory: every .ply / .bin file in it gets its own PNG, named after the
file, in the directory of `--out` (`<stem>.png`; `<name>.png` for clouds that share a stem).

    python -m lidiff_b200.tools.vis_pcd -p results/exp/refine/000123.ply --out view.png
    python -m lidiff_b200.tools.vis_pcd -p results/exp/refine/ --out views/x.png      # views/<scan>.png for every cloud
"""
from __future__ import annotations

import os

import click
import numpy as np

from ..normals import estimate_normals
from ..render import Camera, render, write_png
from .diff_completion_pipeline import load_pcd

CLOUD_SUFFIXES = (".ply", ".bin")


def radius_filter(points: np.ndarray, radius: float) -> np.ndarray:
    """the reference's filter: |p| < radius and -2.5 < z < 3 (radius <= 0: every point)"""
    if radius <= 0.0:
        return points
    dist = np.sum(points ** 2, -1) ** 0.5
    return points[(dist < radius) & (points[:, -1] < 3.0) & (points[:, -1] > -2.5)]


def view(points: np.ndarray, out: str, width=1920, height=1080, point_size=5.0, lookat=None, front=None, up=None, zoom=None) -> str:
    """render `points` with estimated normals from open3d's default camera (overridden by the given values) to the PNG `out`"""
    normals = estimate_normals(points, knn=30) if points.shape[0] else None
    cam = Camera.fit(points, lookat=lookat, front=front, up=up, zoom=zoom, width=width, height=height)
    return write_png(out, render(points, cam, normals=normals, point_size=point_size))


def cloud_files(path: str) -> list[str]:
    if os.path.isdir(path):
        files = sorted(os.path.join(path, f) for f in os.listdir(path) if f.endswith(CLOUD_SUFFIXES))
        if not files:
            raise click.ClickException(f"no .ply or .bin point clouds in {path}")
        return files
    if not os.path.isfile(path):
        raise click.ClickException(f"no such point cloud: {path}")
    return [path]


def png_names(files: list[str]) -> list[str]:
    """<stem>.png per cloud; clouds that share a stem (x.ply and x.bin) keep their suffix (x.ply.png, x.bin.png)"""
    stems = [os.path.splitext(os.path.basename(f))[0] for f in files]
    return [(s if stems.count(s) == 1 else os.path.basename(f)) + ".png" for f, s in zip(files, stems)]


def _vec(v):
    return None if v is None or len(v) == 0 else tuple(v)


@click.command()
@click.option("--path", "-p", type=str, required=True, help="path to pcd (a .ply / .bin file, or a directory of them)")
@click.option("--radius", "-r", type=float, default=50.0, help="range to filter pcd")
@click.option("--out", "-o", type=str, default="view.png", help="PNG to write (for a directory: one PNG per cloud next to it)")
@click.option("--width", type=int, default=1920, help="image width in pixels")
@click.option("--height", type=int, default=1080, help="image height in pixels")
@click.option("--point-size", type=float, default=5.0, help="side of a point's square in pixels")
@click.option("--front", type=float, nargs=3, default=None, help="camera direction from the look-at point to the eye")
@click.option("--lookat", type=float, nargs=3, default=None, help="point the camera looks at (default: the bounding box centre)")
@click.option("--up", type=float, nargs=3, default=None, help="camera up vector")
@click.option("--zoom", type=float, default=None, help="open3d's zoom (default 0.7)")
def main(path, radius, out, width, height, point_size, front, lookat, up, zoom):
    files = cloud_files(path)
    targets = png_names(files) if os.path.isdir(path) else [out]
    for f, target in zip(files, targets):
        if os.path.isdir(path):
            target = os.path.join(os.path.dirname(os.path.abspath(out)), target)
        pts = radius_filter(np.asarray(load_pcd(f), dtype=np.float64), radius)
        try:
            written = view(pts, target, width, height, point_size, _vec(lookat), _vec(front), _vec(up), zoom)
        except ValueError as e:
            raise click.ClickException(str(e))
        click.echo(f"{f}: {pts.shape[0]} points -> {written}")


if __name__ == "__main__":
    main()
