"""ctypes binding of include/lidiff_b200.h (the C-ABI CUDA library, sm_90a).

There is deliberately NO CPU fallback: importing works anywhere (so host logic can be tested), but
`get_lib()` raises if the shared object is missing and `Lib.handle(device)` raises if no H100 (sm_90) is
visible.  torch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_C", "liblidiff_b200.so")

ALGO_AUTO, ALGO_FFMA, ALGO_TC, ALGO_TC_TILE = 0, 1, 2, 3


class Grid(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("vals", C.c_void_p), ("cap_table", C.c_int32)]


class ConvIO(C.Structure):
    _fields_ = [("in1", C.c_void_p), ("in2", C.c_void_p), ("residual", C.c_void_p), ("out", C.c_void_p),
                ("gate_table", C.c_void_p), ("gate_idx", C.c_void_p), ("out_gated", C.c_void_p), ("pre_add", C.c_void_p),
                ("in1_h", C.c_void_p), ("in2_h", C.c_void_p), ("out_h", C.c_void_p), ("out_gated_h", C.c_void_p),
                ("residual_h", C.c_void_p)]


class ConvDesc(C.Structure):
    _fields_ = [("c1", C.c_int32), ("c2", C.c_int32), ("cout", C.c_int32), ("kvol", C.c_int32),
                ("weight", C.c_void_p), ("weight_packed", C.c_void_p),
                ("scale", C.c_void_p), ("shift", C.c_void_p), ("relu", C.c_int32),
                ("nbr", C.c_void_p), ("nbr_stride", C.c_int64),
                ("d_mout", C.c_void_p), ("mout_cap", C.c_int32), ("row_perm", C.c_void_p), ("row_mask", C.c_void_p),
                ("npass", C.c_int32),
                ("io", ConvIO * 2),
                ("tile_order128", C.c_void_p), ("tile_order256", C.c_void_p),
                ("k0", C.c_int32), ("k1", C.c_int32), ("partial_in", C.c_void_p), ("partial_out", C.c_void_p)]


class ScatterDesc(C.Structure):
    _fields_ = [("c1", C.c_int32), ("c2", C.c_int32), ("cout", C.c_int32), ("kvol", C.c_int32),
                ("weight_packed", C.c_void_p), ("pair_in", C.c_void_p), ("pair_out", C.c_void_p),
                ("koff", C.c_void_p), ("tile_off", C.c_void_p), ("npass", C.c_int32),
                ("in1", C.c_void_p * 2), ("in2", C.c_void_p * 2), ("in1_h", C.c_void_p * 2), ("in2_h", C.c_void_p * 2),
                ("out", C.c_void_p * 2),
                ("d_zero_rows", C.c_void_p), ("zero_rows_cap", C.c_int32)]


class DpmCoef(C.Structure):
    _fields_ = [("c_sample", C.c_double), ("c_x0", C.c_double), ("c_noise", C.c_double),
                ("sigma_s", C.c_double), ("alpha_s", C.c_double), ("inv_r0", C.c_double),
                ("guidance_w", C.c_float), ("resolution", C.c_float),
                ("second_order", C.c_int32), ("div_mode", C.c_int32), ("f64_state", C.c_int32)]


EXPORTS = [
    "lb2_create", "lb2_destroy", "lb2_last_error", "lb2_version", "lb2_launch_count", "lb2_read_status",
    "lb2_tile_order", "lb2_row_order_range", "lb2_tile_order_range",
    "lb2_quantize", "lb2_unique_scratch_bytes", "lb2_unique_build", "lb2_voxel_mean_scratch_bytes", "lb2_voxel_mean", "lb2_kernel_map",
    "lb2_spconv_forward", "lb2_packed_weight_bytes", "lb2_pack_weights", "lb2_nn_match", "lb2_linear",
    "lb2_gate_mul", "lb2_gather_rows", "lb2_head_mlp", "lb2_kernel_map_self", "lb2_guidance_dpm_step", "lb2_farthest_point_sample",
    "lb2_row_order", "lb2_row_order_scratch_bytes", "lb2_nn_match_grid",
    "lb2_nn_table_bytes", "lb2_nn_table_build", "lb2_nn_match_table",
    "lb2_nn_tree_bytes", "lb2_nn_tree_build", "lb2_nn_match_tree",
    "lb2_pair_list", "lb2_pair_list_scratch_bytes", "lb2_spconv_scatter", "lb2_spconv_scatter_supported",
    "lb2_pc_tree_bytes", "lb2_pc_nn_scratch_bytes", "lb2_pc_tree_build", "lb2_pc_nn", "lb2_voxel_occupancy", "lb2_occupancy_confusion",
    "lb2_occupancy_bev", "lb2_jsd_scratch_bytes", "lb2_jsd", "lb2_dist_stats_scratch_bytes", "lb2_dist_stats",
    "lb2_map_rehash", "lb2_map_scan_scratch_bytes", "lb2_map_scan",
    "lb2_pc_knn", "lb2_pc_normals", "lb2_fps_batched_capacity", "lb2_farthest_point_sample_batched",
    "lb2_select_points_scratch_bytes", "lb2_select_points", "lb2_viewpoint_filter_scratch_bytes", "lb2_viewpoint_filter",
    "lb2_aggregate_window_scratch_bytes", "lb2_aggregate_window", "lb2_jitter_filter_scratch_bytes", "lb2_jitter_filter",
    "lb2_voxel_first_f64_scratch_bytes", "lb2_voxel_first_f64",
    "lb2_spconv_wgrad_scratch_bytes", "lb2_spconv_wgrad", "lb2_segment_sum",
    "lb2_segment_dot_scratch_bytes", "lb2_segment_dot",
    "lb2_sync_bn_max", "lb2_sync_bn_sum", "lb2_sync_bn_sumsq", "lb2_sync_bn_apply",
    "lb2_sync_bn_backward_max", "lb2_sync_bn_backward_sum", "lb2_sync_bn_backward_apply",
    "lb2_mt19937_words", "lb2_legacy_gauss_scratch_bytes", "lb2_legacy_gauss", "lb2_randperm_scratch_bytes", "lb2_randperm",
    "lb2_render_splat", "lb2_render_shade",
    "lb2_mesh_sample_scratch_bytes", "lb2_mesh_sample_prepare", "lb2_mesh_sample_points",
]

RANGE_NONE, RANGE_FP32, RANGE_FP64 = 0, 1, 2


class Pose(C.Structure):
    _fields_ = [("m", C.c_float * 12)]


class GaussInfo(C.Structure):
    _fields_ = [("words_used", C.c_int64), ("deferred", C.c_int64), ("short_words", C.c_int32), ("has_gauss", C.c_int32),
                ("gauss", C.c_double)]


GAUSS_BAND = 1.0 / 32.0             # LB2_GAUSS_BAND: ulp from a rounding midpoint below which log(r2) is taken from the host's libm
RANDPERM_MAX_N = 214748364          # LB2_RANDPERM_MAX_N = UINT32_MAX // 20


class RenderCamera(C.Structure):
    _fields_ = [("lookat", C.c_double * 3), ("front", C.c_double * 3), ("up", C.c_double * 3), ("distance", C.c_double),
                ("focal", C.c_double), ("width", C.c_int32), ("height", C.c_int32)]


MESH_BAD_INDEX, MESH_NON_FINITE, MESH_BAD_AREA, MESH_BAD_COUNT = 1, 2, 4, 8      # lb2_mesh_info.status bits


class MeshInfo(C.Structure):
    _fields_ = [("surface_area", C.c_double), ("last_count", C.c_int64), ("status", C.c_int32), ("pad", C.c_int32)]


class Segment(C.Structure):
    _fields_ = [("start", C.c_int64), ("m", C.c_double * 12)]


class SelectDesc(C.Structure):
    _fields_ = [("range_mode", C.c_int32), ("center", C.c_double * 3), ("r_min", C.c_double), ("r_max", C.c_double),
                ("has_transform", C.c_int32), ("transform", C.c_double * 12), ("has_z_min", C.c_int32), ("z_min", C.c_double)]


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, int):
        return t
    return t.data_ptr()


class Lib:
    """Loaded shared object + one handle per device."""

    def __init__(self, path: str = _SO):
        if not os.path.exists(path):
            raise RuntimeError(f"lidiff_b200: CUDA library not built ({path}); run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "or lidiff_b200/csrc/build.sh — there is no CPU fallback")
        self.path = path
        self.dll = C.CDLL(path)
        d = self.dll
        d.lb2_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        d.lb2_destroy.argtypes = [C.c_void_p]
        d.lb2_destroy.restype = None
        d.lb2_last_error.argtypes = [C.c_void_p]
        d.lb2_last_error.restype = C.c_char_p
        d.lb2_launch_count.argtypes = [C.c_void_p]
        d.lb2_launch_count.restype = C.c_int64
        d.lb2_read_status.argtypes = [C.c_void_p, C.c_void_p]
        d.lb2_unique_scratch_bytes.argtypes = [C.c_int64]
        d.lb2_unique_scratch_bytes.restype = C.c_size_t
        d.lb2_voxel_mean_scratch_bytes.argtypes = [C.c_int32, C.c_int32]
        d.lb2_voxel_mean_scratch_bytes.restype = C.c_size_t
        d.lb2_packed_weight_bytes.argtypes = [C.c_int32] * 3
        d.lb2_packed_weight_bytes.restype = C.c_size_t
        vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
        d.lb2_quantize.argtypes = [vp, vp, vp, i64, f32, C.c_int, vp]
        d.lb2_unique_build.argtypes = [vp, vp, vp, vp, vp, i32, i32, Grid, vp, vp, vp, vp]
        d.lb2_voxel_mean.argtypes = [vp, vp, vp, vp, i32, i32, vp, i32, vp, vp]
        d.lb2_kernel_map.argtypes = [vp, vp, Grid, vp, vp, i32, i32, i32, vp, i64, vp, vp]
        d.lb2_kernel_map_self.argtypes = [vp, vp, Grid, vp, vp, i32, i32, vp, i64, vp, vp]
        d.lb2_row_order.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, i32]
        d.lb2_tile_order.argtypes = [vp, vp, vp, vp, vp, i32, vp, vp, vp]
        d.lb2_row_order_range.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp, vp, vp]
        d.lb2_tile_order_range.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, vp, vp]
        d.lb2_row_order_scratch_bytes.restype = C.c_size_t
        d.lb2_row_order_scratch_bytes.argtypes = [i32]
        d.lb2_spconv_forward.argtypes = [vp, vp, C.POINTER(ConvDesc), C.c_int]
        d.lb2_pack_weights.argtypes = [vp, vp, vp, i32, i32, i32, vp]
        d.lb2_nn_match.argtypes = [vp, vp, vp, vp, i32, vp, vp, i32, i32, vp]
        d.lb2_pair_list.argtypes = [vp, vp, vp, i64, vp, i32, i32, i32, vp, vp, vp, vp, vp]
        d.lb2_pair_list_scratch_bytes.restype = C.c_size_t
        d.lb2_spconv_scatter.argtypes = [vp, vp, C.POINTER(ScatterDesc)]
        d.lb2_spconv_scatter_supported.argtypes = [i32, i32, i32, i32]
        d.lb2_nn_table_bytes.restype = C.c_size_t
        d.lb2_nn_tree_bytes.restype = C.c_size_t
        d.lb2_nn_tree_bytes.argtypes = [i32]
        d.lb2_nn_tree_build.argtypes = [vp, vp, vp, vp, i32, vp]
        d.lb2_nn_match_tree.argtypes = [vp, vp, vp, vp, i32, vp, i32, vp, vp, vp, vp]
        d.lb2_nn_table_build.argtypes = [vp, vp, vp, vp, i32, vp]
        d.lb2_nn_match_table.argtypes = [vp, vp, vp, vp, i32, vp, vp, i32, vp, i32, i32, vp]
        d.lb2_nn_match_grid.argtypes = [vp, vp, vp, vp, i32, vp, vp, i32, Grid, i32, i32, vp]
        d.lb2_linear.argtypes = [vp, vp, vp, i64, vp, vp, vp, i64, i32, vp, i32, i32, i32, vp, i64,
                                 vp, i32]
        d.lb2_gate_mul.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, vp, vp]
        d.lb2_gather_rows.argtypes = [vp, vp, vp, vp, i32, i32, vp]
        d.lb2_head_mlp.argtypes = [vp, vp, vp, i64, i64, vp, vp, vp, vp, i32, vp, i32, i32, i32, i32, i32, vp, i64, i64]
        d.lb2_guidance_dpm_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, DpmCoef, vp, vp, vp, vp]
        d.lb2_farthest_point_sample.argtypes = [vp, vp, vp, i32, i32, vp, vp]
        d.lb2_fps_batched_capacity.argtypes = [vp]
        d.lb2_fps_batched_capacity.restype = C.c_int64
        d.lb2_farthest_point_sample_batched.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp]
        for f, a in (("lb2_pc_tree_bytes", i32), ("lb2_pc_nn_scratch_bytes", i32), ("lb2_jsd_scratch_bytes", i64),
                     ("lb2_dist_stats_scratch_bytes", i32)):
            getattr(d, f).argtypes = [a]
            getattr(d, f).restype = C.c_size_t
        d.lb2_pc_tree_build.argtypes = [vp, vp, vp, i32, vp]
        d.lb2_pc_nn.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp]
        d.lb2_pc_knn.argtypes = [vp, vp, vp, i32, i32, vp, vp]
        d.lb2_pc_normals.argtypes = [vp, vp, vp, i32, vp, i32, vp]
        d.lb2_voxel_occupancy.argtypes = [vp, vp, vp, i32, vp, i32, vp, vp, vp]
        d.lb2_occupancy_confusion.argtypes = [vp, vp, vp, vp, i64, vp]
        d.lb2_occupancy_bev.argtypes = [vp, vp, vp, i32, vp]
        d.lb2_jsd.argtypes = [vp, vp, vp, vp, i64, vp, vp]
        d.lb2_dist_stats.argtypes = [vp, vp, vp, i32, vp, i32, vp, vp, vp]
        d.lb2_map_rehash.argtypes = [vp, vp, Grid, Grid]
        d.lb2_map_scan_scratch_bytes.argtypes = [i32]
        d.lb2_map_scan_scratch_bytes.restype = C.c_size_t
        d.lb2_map_scan.argtypes = [vp, vp, vp, vp, i32, Pose, f32, i32, Grid, vp, i32, i32, vp, vp]
        d.lb2_select_points_scratch_bytes.argtypes = [i64]
        d.lb2_select_points_scratch_bytes.restype = C.c_size_t
        d.lb2_select_points.argtypes = [vp, vp, vp, i32, i64, i32, vp, C.POINTER(SelectDesc), vp, vp, vp]
        d.lb2_viewpoint_filter_scratch_bytes.argtypes = [i32, i64]
        d.lb2_viewpoint_filter_scratch_bytes.restype = C.c_size_t
        d.lb2_viewpoint_filter.argtypes = [vp, vp, vp, i32, vp, i64, C.c_double, vp, vp, vp]
        f64 = C.c_double
        for f in ("lb2_aggregate_window_scratch_bytes", "lb2_jitter_filter_scratch_bytes", "lb2_voxel_first_f64_scratch_bytes"):
            getattr(d, f).argtypes = [i64]
            getattr(d, f).restype = C.c_size_t
        d.lb2_aggregate_window.argtypes = [vp, vp, vp, vp, i64, vp, i32, C.POINTER(f64), i64, vp, vp, vp]
        d.lb2_jitter_filter.argtypes = [vp, vp, vp, vp, i64, f64, f64, f64, vp, vp, vp]
        d.lb2_voxel_first_f64.argtypes = [vp, vp, vp, i64, f64, f64, vp, vp, vp]
        d.lb2_spconv_wgrad_scratch_bytes.argtypes = [i32, i32, i32, i32]
        d.lb2_spconv_wgrad_scratch_bytes.restype = C.c_size_t
        d.lb2_spconv_wgrad.argtypes = [vp, vp, vp, i32, vp, i32, i32, vp, i64, i32, vp, vp]
        d.lb2_segment_sum.argtypes = [vp, vp, vp, i32, vp, vp, i64, i32, vp]
        d.lb2_segment_dot_scratch_bytes.argtypes = [i64, i32]
        d.lb2_segment_dot_scratch_bytes.restype = C.c_size_t
        d.lb2_segment_dot.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i32, vp, vp]
        d.lb2_sync_bn_max.argtypes = [vp, vp, vp, i64, i32, vp]
        d.lb2_sync_bn_sum.argtypes = [vp, vp, vp, i64, i32, vp, vp]
        d.lb2_sync_bn_sumsq.argtypes = [vp, vp, vp, i64, i32, vp, vp, vp, vp]
        d.lb2_sync_bn_apply.argtypes = [vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp, f64, f64, vp, vp, vp, vp, vp]
        d.lb2_sync_bn_backward_max.argtypes = [vp, vp, vp, vp, i64, i32, vp, vp, vp]
        d.lb2_sync_bn_backward_sum.argtypes = [vp, vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp]
        d.lb2_sync_bn_backward_apply.argtypes = [vp, vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp, vp]
        d.lb2_mt19937_words.argtypes = [vp, vp, vp, i32, i64, vp, C.POINTER(i32)]
        d.lb2_legacy_gauss_scratch_bytes.argtypes = [i64, i64]
        d.lb2_legacy_gauss_scratch_bytes.restype = C.c_size_t
        d.lb2_legacy_gauss.argtypes = [vp, vp, vp, i64, i64, i32, f64, f64, vp, C.POINTER(GaussInfo), vp]
        d.lb2_randperm_scratch_bytes.argtypes = [i64]
        d.lb2_randperm_scratch_bytes.restype = C.c_size_t
        d.lb2_randperm.argtypes = [vp, vp, vp, i64, vp, vp, vp]
        d.lb2_render_splat.argtypes = [vp, vp, vp, i64, C.POINTER(RenderCamera), f64, vp]
        d.lb2_render_shade.argtypes = [vp, vp, vp, vp, vp, vp, f64, f64, C.POINTER(RenderCamera), vp]
        d.lb2_mesh_sample_scratch_bytes.argtypes = [i64]
        d.lb2_mesh_sample_scratch_bytes.restype = C.c_size_t
        d.lb2_mesh_sample_prepare.argtypes = [vp, vp, vp, i64, vp, i64, i64, vp, vp, vp]
        d.lb2_mesh_sample_points.argtypes = [vp, vp, vp, vp, i64, vp, vp, i64, vp]
        self._handles = {}
        self._lock = threading.Lock()

    def missing_symbols(self):
        return [s for s in EXPORTS if not hasattr(self.dll, s)]

    def handle(self, device) -> "Handle":
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("lidiff_b200 runs on CUDA (H100, sm_90a) only; no CPU fallback")
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        with self._lock:
            if idx not in self._handles:
                hp = C.c_void_p()
                rc = self.dll.lb2_create(idx, C.byref(hp))
                if rc != 0:
                    raise RuntimeError(f"lb2_create(device={idx}) failed with {rc} (needs an sm_90 GPU)")
                self._handles[idx] = Handle(self, hp, idx)
            return self._handles[idx]


class Handle:
    def __init__(self, lib: Lib, hp, device_index: int):
        self.lib, self.dll, self.hp, self.device_index = lib, lib.dll, hp, device_index
        self.device = torch.device("cuda", device_index)

    # -- plumbing ----------------------------------------------------------------------------------
    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _check(self, rc, what):
        if rc != 0:
            msg = self.dll.lb2_last_error(self.hp)
            raise RuntimeError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")

    def launch_count(self) -> int:
        return int(self.dll.lb2_launch_count(self.hp))

    def read_status(self) -> int:
        return int(self.dll.lb2_read_status(self.hp, self._stream()))

    # -- coordinate manager ------------------------------------------------------------------------
    def new_grid(self, n_cap: int):
        cap = 1 << max(4, (2 * n_cap - 1).bit_length())
        keys = torch.empty(cap, dtype=torch.int64, device=self.device)
        vals = torch.empty(2 * cap, dtype=torch.int32, device=self.device)
        return (keys, vals, cap)

    @staticmethod
    def _grid(g):
        return Grid(g[0].data_ptr(), g[1].data_ptr(), g[2])

    def unique_scratch(self, n_cap: int) -> torch.Tensor:
        nbytes = int(self.dll.lb2_unique_scratch_bytes(n_cap))
        return torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    def quantize(self, x, resolution, div_mode, out):
        self._check(self.dll.lb2_quantize(self.hp, self._stream(), _ptr(x), x.numel(), float(resolution), int(div_mode), _ptr(out)), "lb2_quantize")

    def unique_build(self, in_f, in_i, d_nin, n_cap, ts_floor, grid, out_coords, inverse, d_nout, scratch):
        self._check(self.dll.lb2_unique_build(self.hp, self._stream(), _ptr(in_f), _ptr(in_i), _ptr(d_nin), int(n_cap), int(ts_floor),
                                              self._grid(grid), _ptr(out_coords), _ptr(inverse), _ptr(d_nout), _ptr(scratch)), "lb2_unique_build")

    def voxel_mean_scratch(self, m_cap: int, c: int) -> torch.Tensor:
        nbytes = int(self.dll.lb2_voxel_mean_scratch_bytes(int(m_cap), int(c)))
        return torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    def voxel_mean(self, feats, inverse, n, c, d_m, m_cap, out, scratch):
        self._check(self.dll.lb2_voxel_mean(self.hp, self._stream(), _ptr(feats), _ptr(inverse), int(n), int(c), _ptr(d_m), int(m_cap),
                                            _ptr(out), _ptr(scratch)), "lb2_voxel_mean")

    def kernel_map(self, grid_in, out_coords, d_nout, nout_cap, ks, step, nbr, nbr_stride, pair_count=None, row_mask=None):
        self._check(self.dll.lb2_kernel_map(self.hp, self._stream(), self._grid(grid_in), _ptr(out_coords), _ptr(d_nout), int(nout_cap),
                                            int(ks), int(step), _ptr(nbr), int(nbr_stride), _ptr(pair_count), _ptr(row_mask)), "lb2_kernel_map")

    def kernel_map_self(self, grid, coords, d_n, n_cap, step, nbr, nbr_stride, pair_count=None, row_mask=None):
        self._check(self.dll.lb2_kernel_map_self(self.hp, self._stream(), self._grid(grid), _ptr(coords), _ptr(d_n), int(n_cap), int(step),
                                                 _ptr(nbr), int(nbr_stride), _ptr(pair_count), _ptr(row_mask)), "lb2_kernel_map_self")

    def row_order_scratch_bytes(self, n_cap) -> int:
        return int(self.dll.lb2_row_order_scratch_bytes(int(n_cap)))

    def row_order(self, row_mask, d_n, n_cap, kvol, perm, scratch, coords=None, coord_shift=0):
        self._check(self.dll.lb2_row_order(self.hp, self._stream(), _ptr(row_mask), _ptr(d_n), int(n_cap), int(kvol), _ptr(perm), _ptr(scratch),
                                           _ptr(coords), int(coord_shift)), "lb2_row_order")

    def tile_order(self, row_mask, row_perm, d_n, n_cap, order128, order256, scratch):
        self._check(self.dll.lb2_tile_order(self.hp, self._stream(), _ptr(row_mask), _ptr(row_perm), _ptr(d_n), int(n_cap), _ptr(order128),
                                            _ptr(order256), _ptr(scratch)), "lb2_tile_order")

    def row_order_range(self, row_mask, d_n, n_cap, k0, k1, perm, d_live, scratch):
        self._check(self.dll.lb2_row_order_range(self.hp, self._stream(), _ptr(row_mask), _ptr(d_n), int(n_cap), int(k0), int(k1), _ptr(perm),
                                                 _ptr(d_live), _ptr(scratch)), "lb2_row_order_range")

    def tile_order_range(self, row_mask, row_perm, d_n, n_cap, k0, k1, order128, scratch):
        self._check(self.dll.lb2_tile_order_range(self.hp, self._stream(), _ptr(row_mask), _ptr(row_perm), _ptr(d_n), int(n_cap), int(k0), int(k1),
                                                  _ptr(order128), _ptr(scratch)), "lb2_tile_order_range")

    # -- conv ----------------------------------------------------------------------------------------
    def spconv(self, desc: ConvDesc, algo: int = ALGO_AUTO):
        self._check(self.dll.lb2_spconv_forward(self.hp, self._stream(), C.byref(desc), int(algo)), "lb2_spconv_forward")

    def pair_list(self, nbr, nbr_stride, d_nout, nout_cap, kvol, skip_k, pair_in, pair_out, koff, tile_off, scratch):
        self._check(self.dll.lb2_pair_list(self.hp, self._stream(), _ptr(nbr), int(nbr_stride), _ptr(d_nout), int(nout_cap), int(kvol), int(skip_k),
                                           _ptr(pair_in), _ptr(pair_out), _ptr(koff), _ptr(tile_off), _ptr(scratch)), "lb2_pair_list")

    def scatter_supported(self, c1, c2, cout, kvol) -> bool:
        return bool(self.dll.lb2_spconv_scatter_supported(int(c1), int(c2), int(cout), int(kvol)))

    def spconv_scatter(self, desc: "ScatterDesc"):
        self._check(self.dll.lb2_spconv_scatter(self.hp, self._stream(), C.byref(desc)), "lb2_spconv_scatter")

    def packed_weight_bytes(self, kvol, cin, cout) -> int:
        return int(self.dll.lb2_packed_weight_bytes(kvol, cin, cout))

    def pack_weights(self, w: torch.Tensor):
        kvol, cin, cout = w.shape
        nbytes = self.packed_weight_bytes(kvol, cin, cout)
        if nbytes == 0:
            return None
        out = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self._check(self.dll.lb2_pack_weights(self.hp, self._stream(), _ptr(w), kvol, cin, cout, _ptr(out)), "lb2_pack_weights")
        return out

    def spconv_wgrad(self, x, g, nbr, kvol, dw):
        """dw (kvol, cin, cout) fp32 = per offset k: sum over output rows o of x[nbr[k][o]]^T g[o] (nbr None: identity, kvol 1)"""
        cin, (m_out, cout) = x.shape[1], g.shape
        nbytes = int(self.dll.lb2_spconv_wgrad_scratch_bytes(int(kvol), int(cin), int(cout), int(m_out)))
        if nbytes == 0:
            raise RuntimeError(f"lb2_spconv_wgrad: no kernel for kvol {kvol}, {cin} -> {cout} channels")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self._check(self.dll.lb2_spconv_wgrad(self.hp, self._stream(), _ptr(x), int(cin), _ptr(g), int(cout), int(m_out), _ptr(nbr),
                                              int(nbr.stride(0)) if nbr is not None else 0, int(kvol), _ptr(dw), _ptr(scratch)),
                    "lb2_spconv_wgrad")

    def segment_sum(self, values, order, offsets, out):
        """out[s] = sum of values[order[i]] over i in [offsets[s], offsets[s + 1]), in ascending i (order None: identity)"""
        self._check(self.dll.lb2_segment_sum(self.hp, self._stream(), _ptr(values), int(values.dtype == torch.float64), _ptr(order),
                                             _ptr(offsets), int(offsets.shape[0] - 1), int(values.shape[1]), _ptr(out)), "lb2_segment_sum")

    def segment_dot(self, a, b, order, offsets, out):
        """out[s] = sum of a[order[i]] * b[order[i]] over i in [offsets[s], offsets[s + 1]) in lb2_segment_dot's chunked order (b None:
        of a[order[i]]); a, b (rows, c) fp32, order int64 over every row"""
        if a.dtype != torch.float32 or (b is not None and b.dtype != torch.float32):
            raise RuntimeError("lb2_segment_dot: fp32 operands only")
        nrows, c = (a.shape[0] if order is None else order.shape[0]), a.shape[1]
        scratch = torch.empty(int(self.dll.lb2_segment_dot_scratch_bytes(int(nrows), int(c))), dtype=torch.uint8, device=self.device)
        self._check(self.dll.lb2_segment_dot(self.hp, self._stream(), _ptr(a), _ptr(b), _ptr(order), _ptr(offsets), int(nrows),
                                             int(offsets.shape[0] - 1), int(c), _ptr(out), _ptr(scratch)), "lb2_segment_dot")

    # -- synchronised batch norm (include/lidiff_b200.h: the words, formulas and the collective between each call) ---------------
    def sync_bn_max(self, x, max_words):
        """max_words int64 (2c,): per channel the largest finite |x| (fp32 bits) and a non-finite flag; combine with MAX"""
        n, c = x.shape
        self._check(self.dll.lb2_sync_bn_max(self.hp, self._stream(), _ptr(x), int(n), int(c), _ptr(max_words)), "lb2_sync_bn_max")

    def sync_bn_sum(self, x, max_words, sum_words):
        """sum_words int64 (2c + 1,): the fixed-point sum of x per channel and the row count; combine with SUM"""
        n, c = x.shape
        self._check(self.dll.lb2_sync_bn_sum(self.hp, self._stream(), _ptr(x), int(n), int(c), _ptr(max_words), _ptr(sum_words)),
                    "lb2_sync_bn_sum")

    def sync_bn_sumsq(self, x, max_words, sum_words, mean, sq_words):
        """mean fp64 (c,) from the combined sums; sq_words int64 (4c,): the fixed-point sum of (x - mean)^2; combine with SUM"""
        n, c = x.shape
        self._check(self.dll.lb2_sync_bn_sumsq(self.hp, self._stream(), _ptr(x), int(n), int(c), _ptr(max_words), _ptr(sum_words),
                                               _ptr(mean), _ptr(sq_words)), "lb2_sync_bn_sumsq")

    def sync_bn_apply(self, x, max_words, sum_words, mean, sq_words, gamma, beta, eps, momentum, running_mean, running_var, var, invstd,
                      y):
        """var, invstd fp64 (c,), the running statistics (None: not tracked) and y = the normalised x"""
        n, c = x.shape
        self._check(self.dll.lb2_sync_bn_apply(self.hp, self._stream(), _ptr(x), int(n), int(c), _ptr(max_words), _ptr(sum_words), _ptr(mean),
                                               _ptr(sq_words), _ptr(gamma), _ptr(beta), float(eps), float(momentum), _ptr(running_mean),
                                               _ptr(running_var), _ptr(var), _ptr(invstd), _ptr(y)), "lb2_sync_bn_apply")

    def sync_bn_backward_max(self, dy, x, mean, invstd, max_words):
        """max_words int64 (3c,): the largest finite |dy| and |dy xhat| and a non-finite flag per channel; combine with MAX"""
        n, c = x.shape
        self._check(self.dll.lb2_sync_bn_backward_max(self.hp, self._stream(), _ptr(dy), _ptr(x), int(n), int(c), _ptr(mean), _ptr(invstd),
                                                      _ptr(max_words)), "lb2_sync_bn_backward_max")

    def sync_bn_backward_sum(self, dy, x, mean, invstd, max_words, sum_words, dgamma, dbeta):
        """sum_words int64 (4c,): the fixed-point sums of dy and dy xhat (combine with SUM); dgamma / dbeta: this rank's sums"""
        n, c = x.shape
        self._check(self.dll.lb2_sync_bn_backward_sum(self.hp, self._stream(), _ptr(dy), _ptr(x), int(n), int(c), _ptr(mean), _ptr(invstd),
                                                      _ptr(max_words), _ptr(sum_words), _ptr(dgamma), _ptr(dbeta)),
                    "lb2_sync_bn_backward_sum")

    def sync_bn_backward_apply(self, dy, x, mean, invstd, gamma, max_words, sum_words, count, dx):
        """dx from the combined backward sums; count = the forward's combined sum_words[2c:]"""
        n, c = x.shape
        self._check(self.dll.lb2_sync_bn_backward_apply(self.hp, self._stream(), _ptr(dy), _ptr(x), int(n), int(c), _ptr(mean), _ptr(invstd),
                                                        _ptr(gamma), _ptr(max_words), _ptr(sum_words), _ptr(count), _ptr(dx)),
                    "lb2_sync_bn_backward_apply")

    # -- misc ----------------------------------------------------------------------------------------
    def nn_match(self, q, d_nq, nq_cap, k, d_nk, nk_cap, batch_scale, idx):
        self._check(self.dll.lb2_nn_match(self.hp, self._stream(), _ptr(q), _ptr(d_nq), int(nq_cap), _ptr(k), _ptr(d_nk), int(nk_cap),
                                          int(batch_scale), _ptr(idx)), "lb2_nn_match")

    def nn_match_grid(self, q, d_nq, nq_cap, k, d_nk, nk_cap, key_grid, key_stride, max_ring, idx):
        self._check(self.dll.lb2_nn_match_grid(self.hp, self._stream(), _ptr(q), _ptr(d_nq), int(nq_cap), _ptr(k), _ptr(d_nk), int(nk_cap),
                                               self._grid(key_grid), int(key_stride), int(max_ring), _ptr(idx)), "lb2_nn_match_grid")

    def nn_table(self, k, d_nk, nk_cap):
        """compact hash table of the key voxels for nn_match_table (one per conditioning scan)"""
        t = torch.empty(int(self.dll.lb2_nn_table_bytes()), dtype=torch.uint8, device=self.device)
        self._check(self.dll.lb2_nn_table_build(self.hp, self._stream(), _ptr(k), _ptr(d_nk), int(nk_cap), _ptr(t)), "lb2_nn_table_build")
        return t

    def nn_tree(self, k, d_nk, nk_cap, out=None):
        """bounding-box hierarchy over the key voxels for nn_match_tree (one per conditioning scan); `out` re-uses a buffer"""
        nbytes = int(self.dll.lb2_nn_tree_bytes(int(nk_cap)))
        t = out if (out is not None and out.numel() == nbytes) else torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self._check(self.dll.lb2_nn_tree_build(self.hp, self._stream(), _ptr(k), _ptr(d_nk), int(nk_cap), _ptr(t)), "lb2_nn_tree_build")
        return t

    def nn_match_tree(self, q, d_nq, nq_cap, tree, nk_cap, idx, k=None, hint_of=None, hint_idx=None):
        self._check(self.dll.lb2_nn_match_tree(self.hp, self._stream(), _ptr(q), _ptr(d_nq), int(nq_cap), _ptr(tree), int(nk_cap),
                                               _ptr(k), _ptr(hint_of), _ptr(hint_idx), _ptr(idx)), "lb2_nn_match_tree")

    def nn_match_table(self, q, d_nq, nq_cap, k, d_nk, nk_cap, table, key_stride, max_ring, idx):
        self._check(self.dll.lb2_nn_match_table(self.hp, self._stream(), _ptr(q), _ptr(d_nq), int(nq_cap), _ptr(k), _ptr(d_nk), int(nk_cap),
                                                _ptr(table), int(key_stride), int(max_ring), _ptr(idx)), "lb2_nn_match_table")

    def linear(self, x, ldx, w, b, addend, ld_add, m_cap, d_m, n_in, n_out, act, y, ldy, prebias=None, pre_act=0):
        self._check(self.dll.lb2_linear(self.hp, self._stream(), _ptr(x), int(ldx), _ptr(w), _ptr(b), _ptr(addend), int(ld_add), int(m_cap),
                                        _ptr(d_m), int(n_in), int(n_out), int(act), _ptr(y), int(ldy), _ptr(prebias), int(pre_act)), "lb2_linear")

    def head_mlp(self, x, ldx, x_pass_stride, w0, b0, w1, b1, m_cap, d_m, n_in, n_hid, n_out, out_act, npass, y, ldy, y_pass_stride):
        self._check(self.dll.lb2_head_mlp(self.hp, self._stream(), _ptr(x), int(ldx), int(x_pass_stride), _ptr(w0), _ptr(b0), _ptr(w1), _ptr(b1),
                                          int(m_cap), _ptr(d_m), int(n_in), int(n_hid), int(n_out), int(out_act), int(npass), _ptr(y), int(ldy),
                                          int(y_pass_stride)), "lb2_head_mlp")

    def gate_mul(self, x, table, idx, d_m, m_cap, c, out, out_h=None):
        self._check(self.dll.lb2_gate_mul(self.hp, self._stream(), _ptr(x), _ptr(table), _ptr(idx), _ptr(d_m), int(m_cap), int(c), _ptr(out),
                                          _ptr(out_h)), "lb2_gate_mul")

    def gather_rows(self, src, idx, n, c, out):
        self._check(self.dll.lb2_gather_rows(self.hp, self._stream(), _ptr(src), _ptr(idx), int(n), int(c), _ptr(out)), "lb2_gather_rows")

    def guidance_dpm_step(self, eps_c, eps_u, inverse, x_t, x_init, noise, x0_state, n_points, coef: DpmCoef,
                          eps_out, x_next, coord_next, batch_col=None):
        self._check(self.dll.lb2_guidance_dpm_step(self.hp, self._stream(), _ptr(eps_c), _ptr(eps_u), _ptr(inverse), _ptr(x_t), _ptr(x_init),
                                                   _ptr(noise), _ptr(x0_state), int(n_points), coef, _ptr(eps_out), _ptr(x_next),
                                                   _ptr(coord_next), _ptr(batch_col)), "lb2_guidance_dpm_step")

    def farthest_point_sample(self, pts, n, n_samples, out_idx, dist):
        self._check(self.dll.lb2_farthest_point_sample(self.hp, self._stream(), _ptr(pts), int(n), int(n_samples), _ptr(out_idx), _ptr(dist)),
                    "lb2_farthest_point_sample")

    def fps_batched_capacity(self) -> int:
        """most points a scan may have in farthest_point_sample_batched (0: the device cannot run its cluster)"""
        return int(self.dll.lb2_fps_batched_capacity(self.hp))

    def farthest_point_sample_batched(self, pts, offsets, n_scans, max_n, n_samples, out_idx):
        self._check(self.dll.lb2_farthest_point_sample_batched(self.hp, self._stream(), _ptr(pts), _ptr(offsets), int(n_scans), int(max_n),
                                                               int(n_samples), _ptr(out_idx)), "lb2_farthest_point_sample_batched")

    # -- evaluation metrics (fp64 (n, 3) contiguous point tensors) ---------------------------------------------------------------
    def _bytes(self, nbytes):
        return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=self.device)

    def pc_tree(self, pts):
        """Morton-sorted box hierarchy over the reference cloud `pts` for pc_nn"""
        n = pts.shape[0]
        tree = self._bytes(self.dll.lb2_pc_tree_bytes(n))
        self._check(self.dll.lb2_pc_tree_build(self.hp, self._stream(), _ptr(pts), int(n), _ptr(tree)), "lb2_pc_tree_build")
        return tree

    def pc_nn(self, q, tree, dist, idx=None):
        """dist[i] = distance of q[i] to its nearest point of the tree's cloud; idx[i] = that point (lowest index on ties)"""
        nq = q.shape[0]
        scratch = self._bytes(self.dll.lb2_pc_nn_scratch_bytes(nq))
        self._check(self.dll.lb2_pc_nn(self.hp, self._stream(), _ptr(q), int(nq), _ptr(tree), _ptr(dist), _ptr(idx), _ptr(scratch)),
                    "lb2_pc_nn")

    def pc_knn(self, tree, n, k, idx, d2=None):
        """idx (n, min(k, n)) int32 = the nearest points of each of the tree's n points, itself included, in (d², index) order;
        d2 the same shape fp64 (optional); 1 <= k <= 32"""
        self._check(self.dll.lb2_pc_knn(self.hp, self._stream(), _ptr(tree), int(n), int(k), _ptr(idx), _ptr(d2)), "lb2_pc_knn")

    def pc_normals(self, pts, idx, normals):
        """normals (n, 3) fp64 = open3d FastEigen3x3 normal of the cumulant covariance of each row of `idx` (n, k) int32"""
        n, k = idx.shape
        self._check(self.dll.lb2_pc_normals(self.hp, self._stream(), _ptr(pts), int(n), _ptr(idx), int(k), _ptr(normals)), "lb2_pc_normals")

    def voxel_occupancy(self, pts, edges, bits=None, counts=None, n_in=None):
        bins = edges.shape[0] - 1
        self._check(self.dll.lb2_voxel_occupancy(self.hp, self._stream(), _ptr(pts), int(pts.shape[0]), _ptr(edges), int(bins), _ptr(bits),
                                                 _ptr(counts), _ptr(n_in)), "lb2_voxel_occupancy")

    def occupancy_confusion(self, bits_gt, bits_pred, nbits, out):
        self._check(self.dll.lb2_occupancy_confusion(self.hp, self._stream(), _ptr(bits_gt), _ptr(bits_pred), int(nbits), _ptr(out)),
                    "lb2_occupancy_confusion")

    def occupancy_bev(self, bits, bins, bev):
        self._check(self.dll.lb2_occupancy_bev(self.hp, self._stream(), _ptr(bits), int(bins), _ptr(bev)), "lb2_occupancy_bev")

    def jsd(self, hist_a, hist_b, out):
        n = hist_a.numel()
        scratch = self._bytes(self.dll.lb2_jsd_scratch_bytes(n))
        self._check(self.dll.lb2_jsd(self.hp, self._stream(), _ptr(hist_a), _ptr(hist_b), int(n), _ptr(out), _ptr(scratch)), "lb2_jsd")

    def dist_stats(self, dist, thresholds, sum_out, counts_out):
        nt = thresholds.shape[0]
        scratch = self._bytes(self.dll.lb2_dist_stats_scratch_bytes(nt))
        self._check(self.dll.lb2_dist_stats(self.hp, self._stream(), _ptr(dist), int(dist.shape[0]), _ptr(thresholds), int(nt), _ptr(sum_out),
                                            _ptr(counts_out), _ptr(scratch)), "lb2_dist_stats")

    # -- ground-truth maps (lidiff_b200.maps) -------------------------------------------------------------------------------------
    def new_map_table(self, cap: int):
        """an empty voxel-key table of `cap` (a power of two) slots, in new_grid's (keys, vals, cap) form"""
        return (torch.empty(cap, dtype=torch.int64, device=self.device), torch.empty(2 * cap, dtype=torch.int32, device=self.device), cap)

    def map_rehash(self, old, table):
        """clear `table` and insert the (key, row) pairs of `old` (None: none)"""
        self._check(self.dll.lb2_map_rehash(self.hp, self._stream(), self._grid(old) if old is not None else Grid(None, None, 0),
                                            self._grid(table)), "lb2_map_rehash")

    def map_scan_scratch(self, n_cap: int) -> torch.Tensor:
        return self._bytes(self.dll.lb2_map_scan_scratch_bytes(int(n_cap)))

    def map_scan(self, points, labels, pose12, voxel_size, div_mode, table, map_buf, map_n, out, scratch):
        """filter, transform and insert the (n, 4) `points` (int32 / uint32 `labels` or None); out[0] = new rows appended to
        map_buf[map_n:], out[1] = status (bit0: voxel index outside the key range)"""
        pose = Pose((C.c_float * 12)(*[float(v) for v in pose12]))
        self._check(self.dll.lb2_map_scan(self.hp, self._stream(), _ptr(points), _ptr(labels), int(points.shape[0]), pose, float(voxel_size),
                                          int(div_mode), self._grid(table), _ptr(map_buf), int(map_n), int(map_buf.shape[0]), _ptr(out),
                                          _ptr(scratch)), "lb2_map_scan")

    # -- training / test samples (lidiff_b200.datasets) ---------------------------------------------------------------------------
    def select_points_scratch(self, n: int) -> torch.Tensor:
        return self._bytes(self.dll.lb2_select_points_scratch_bytes(int(n)))

    def select_points(self, points, labels, desc: SelectDesc, out, d_count, scratch):
        """order-preserving filter + transform of the (n, 3 | 4) fp32 / fp64 rows `points` (uint32 / int32 `labels` or None) into the
        fp64 (>= n, 3) `out`; d_count[0] = rows kept"""
        n, stride = points.shape
        self._check(self.dll.lb2_select_points(self.hp, self._stream(), _ptr(points), int(points.dtype == torch.float64), int(n),
                                               int(stride), _ptr(labels), C.byref(desc), _ptr(out), _ptr(d_count), _ptr(scratch)),
                    "lb2_select_points")

    def viewpoint_filter_scratch(self, n_part: int, n_full: int) -> torch.Tensor:
        return self._bytes(self.dll.lb2_viewpoint_filter_scratch_bytes(int(n_part), int(n_full)))

    def viewpoint_filter(self, part, full, voxel_size, out, d_out, scratch):
        """rows of the fp64 (n, 3) `full` whose voxel_size cell holds a row of `part` -> `out` in order; d_out = [rows, status]"""
        self._check(self.dll.lb2_viewpoint_filter(self.hp, self._stream(), _ptr(part), int(part.shape[0]), _ptr(full), int(full.shape[0]),
                                                  float(voxel_size), _ptr(out), _ptr(d_out), _ptr(scratch)), "lb2_viewpoint_filter")

    # -- refinement samples (lidiff_b200.datasets_refine) -------------------------------------------------------------------------
    def aggregate_window_scratch(self, n: int) -> torch.Tensor:
        return self._bytes(self.dll.lb2_aggregate_window_scratch_bytes(int(n)))

    def aggregate_window(self, points, labels, segments, nseg, undo12, split, out, d_out, scratch):
        """label / range filter and the two rigid transforms of the window's (n, 4) fp32 `points` (int32 / uint32 `labels`) into the
        fp64 (>= n, 3) `out`; `segments` = a device byte tensor of nseg Segment records; d_out = [rows kept, rows kept before `split`]"""
        undo = (C.c_double * 12)(*[float(v) for v in undo12])
        self._check(self.dll.lb2_aggregate_window(self.hp, self._stream(), _ptr(points), _ptr(labels), int(points.shape[0]), _ptr(segments),
                                                  int(nseg), undo, int(split), _ptr(out), _ptr(d_out), _ptr(scratch)),
                    "lb2_aggregate_window")

    def jitter_filter_scratch(self, n: int) -> torch.Tensor:
        return self._bytes(self.dll.lb2_jitter_filter_scratch_bytes(int(n)))

    def jitter_filter(self, points, randn, sigma, clip, max_range, out, d_count, scratch):
        """rows p + clip(sigma * randn, +-clip) of the fp64 (n, 3) `points` within max_range -> `out` in order; d_count[0] = rows"""
        self._check(self.dll.lb2_jitter_filter(self.hp, self._stream(), _ptr(points), _ptr(randn), int(points.shape[0]), float(sigma),
                                               float(clip), float(max_range), _ptr(out), _ptr(d_count), _ptr(scratch)), "lb2_jitter_filter")

    def voxel_first_f64_scratch(self, n: int) -> torch.Tensor:
        return self._bytes(self.dll.lb2_voxel_first_f64_scratch_bytes(int(n)))

    def voxel_first_f64(self, points, voxel_size, max_range, out, d_out, scratch):
        """first row of every floor(p / voxel_size) voxel of the fp64 (n, 3) `points`, within max_range -> `out` in row order;
        d_out = [rows, status]"""
        self._check(self.dll.lb2_voxel_first_f64(self.hp, self._stream(), _ptr(points), int(points.shape[0]), float(voxel_size),
                                                 float(max_range), _ptr(out), _ptr(d_out), _ptr(scratch)), "lb2_voxel_first_f64")

    # -- host random streams on the device (lidiff_b200.rng) ----------------------------------------------------------------------
    def mt19937_words(self, state, pos, n, out) -> int:
        """out[:n] = the next n tempered MT19937 words of `state` (device int32 (624,), updated in place) at numpy position `pos`;
        returns the position afterwards"""
        pos_out = C.c_int32()
        self._check(self.dll.lb2_mt19937_words(self.hp, self._stream(), _ptr(state), int(pos), int(n), _ptr(out), C.byref(pos_out)),
                    "lb2_mt19937_words")
        return int(pos_out.value)

    def legacy_gauss(self, words, n_words, n_out, has_gauss, gauss, band, out) -> GaussInfo:
        """numpy's legacy_gauss n_out times over the first n_words of `words` -> out (fp64); synchronises the stream"""
        info = GaussInfo()
        scratch = self._bytes(self.dll.lb2_legacy_gauss_scratch_bytes(int(n_words), int(n_out)))
        self._check(self.dll.lb2_legacy_gauss(self.hp, self._stream(), _ptr(words), int(n_words), int(n_out), int(has_gauss), float(gauss),
                                              float(band), _ptr(out), C.byref(info), _ptr(scratch)), "lb2_legacy_gauss")
        return info

    def randperm(self, words, n, out, d_rounds=None):
        """out (int64 (n,)) = torch's CPU randperm(n) shuffle driven by the n - 1 words `words`"""
        scratch = self._bytes(self.dll.lb2_randperm_scratch_bytes(int(n)))
        self._check(self.dll.lb2_randperm(self.hp, self._stream(), _ptr(words), int(n), _ptr(out), _ptr(d_rounds), _ptr(scratch)),
                    "lb2_randperm")

    # -- point-cloud images (lidiff_b200.render) ----------------------------------------------------------------------------------
    def render_splat(self, pts, cam: RenderCamera, point_size, keys):
        """keys (uint64 as int64 (height width,), filled with -1 first) <- atomicMin of (float depth bits << 32 | index) over the
        pixels each point of the fp64 (n, 3) `pts` covers"""
        self._check(self.dll.lb2_render_splat(self.hp, self._stream(), _ptr(pts), int(pts.shape[0]), C.byref(cam), float(point_size),
                                              _ptr(keys)), "lb2_render_splat")

    def render_shade(self, keys, pts, normals, colors, z_lo, z_hi, cam: RenderCamera, rgb):
        """rgb (uint8 (height, width, 3)) from the keys: white background, colours or jet of z, the headlight of the normals"""
        self._check(self.dll.lb2_render_shade(self.hp, self._stream(), _ptr(keys), _ptr(pts), _ptr(normals), _ptr(colors), float(z_lo),
                                              float(z_hi), C.byref(cam), _ptr(rgb)), "lb2_render_shade")

    # -- uniform surface sampling of triangle meshes (lidiff_b200.mesh) -----------------------------------------------------------
    def mesh_sample_scratch(self, n_tris: int) -> torch.Tensor:
        return self._bytes(self.dll.lb2_mesh_sample_scratch_bytes(int(n_tris)))

    def mesh_sample_prepare(self, verts, tris, n_points, area, info, scratch):
        """area (fp64 (n_tris,)), S and the status into `info` (a device byte tensor of sizeof(MeshInfo)), the points' triangle
        bounds n_t into `scratch`, for the fp64 (n_verts, 3) `verts` and int32 (n_tris, 3) `tris`"""
        self._check(self.dll.lb2_mesh_sample_prepare(self.hp, self._stream(), _ptr(verts), int(verts.shape[0]), _ptr(tris), int(tris.shape[0]),
                                                     int(n_points), _ptr(area), _ptr(info), _ptr(scratch)), "lb2_mesh_sample_prepare")

    def mesh_sample_points(self, verts, tris, scratch, words, n_points, out):
        """out (fp64 (n_points, 3)) from a clean mesh_sample_prepare and the 4 n_points MT19937 words `words`"""
        self._check(self.dll.lb2_mesh_sample_points(self.hp, self._stream(), _ptr(verts), _ptr(tris), int(tris.shape[0]), _ptr(scratch),
                                                    _ptr(words), int(n_points), _ptr(out)), "lb2_mesh_sample_points")


_LIB = None


def get_lib() -> Lib:
    global _LIB
    if _LIB is None:
        _LIB = Lib()
    return _LIB


def get_handle(device) -> Handle:
    return get_lib().handle(device)
