"""TEST INFRASTRUCTURE: CPU stand-ins for the rendering methods of `lidiff_b200._lib.Handle` (render_splat, render_shade), computed
by the numpy restatement of tests/render_reference.py, on top of the normal stand-ins of tests/fake_normals_backend.py, so the host
logic of lidiff_b200.render, the vis_pcd CLI and the open3d shim's draw_geometries can be exercised without a GPU.  Tests install
it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_normals_backend
import render_reference


class _Cam:
    """the fields of an lb2_render_camera, as the restatement reads them"""

    def __init__(self, c):
        self.lookat, self.front, self.up = tuple(c.lookat), tuple(c.front), tuple(c.up)
        self.distance, self.focal, self.width, self.height = c.distance, c.focal, c.width, c.height


class FakeRenderHandle(fake_normals_backend.FakeNormalsHandle):
    def render_splat(self, pts, cam, point_size, keys):
        assert pts.dtype == torch.float64 and keys.dtype == torch.int64 and keys.shape[0] == cam.width * cam.height
        self.launches += 1
        k = keys.numpy().view(np.uint64)
        render_reference.splat(pts.numpy(), _Cam(cam), point_size, keys=k)

    def render_shade(self, keys, pts, normals, colors, z_lo, z_hi, cam, rgb):
        assert rgb.dtype == torch.uint8 and tuple(rgb.shape) == (cam.height, cam.width, 3)
        self.launches += 1
        out = render_reference.shade(keys.numpy().view(np.uint64), pts.numpy(), _Cam(cam),
                                     None if normals is None else normals.numpy(), None if colors is None else colors.numpy(), z_lo, z_hi)
        rgb[:] = torch.from_numpy(out)


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake with the rendering stand-ins (host-logic tests only)"""
    from lidiff_b200 import _lib
    h = FakeRenderHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
