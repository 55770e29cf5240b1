"""Oracle: MinkowskiEngine-0.5.4 operator semantics restated on CPU (torch / numpy).

TEST INFRASTRUCTURE — see `oracle/__init__.py`.  Every function cites the reference
call site whose behaviour it stands for (paths relative to /root/reference) and the
SURVEY.md appendix that specifies the third-party semantics.

Row-order convention (SURVEY.md App. A.9): level-0 rows in first-occurrence order of
the input points; coarser levels in first-occurrence order over the parent's rows.
"""
from __future__ import annotations

import numpy as np
import torch

# ----------------------------------------------------------------------------------------------
# coordinate packing: [b | x | y | z] -> one int64 so numpy can unique / searchsorted on it.
# 10 bits batch (0..1023), 18 bits two's complement per axis: [-131072, 131071] voxels (+-6.5 km at
# 5 cm), a range the stride levels' floor to multiples of 2^l never leaves.
# The CUDA hash grid uses the same packing (lidiff_b200/csrc/common.cuh).
# ----------------------------------------------------------------------------------------------
AXIS_BITS = 18
AXIS_OFF = 1 << (AXIS_BITS - 1)
BATCH_MAX = 1 << 10


def in_key_range(xyz: np.ndarray) -> np.ndarray:
    """(..., 3) integer axes -> bool (...): every axis in [-AXIS_OFF, AXIS_OFF)"""
    return ((xyz >= -AXIS_OFF) & (xyz < AXIS_OFF)).all(-1)


def pack_keys(C: np.ndarray) -> np.ndarray:
    C = np.asarray(C, dtype=np.int64)
    if C.shape[0]:
        assert C[:, 0].min() >= 0 and C[:, 0].max() < BATCH_MAX, "batch index out of key range"
        assert in_key_range(C[:, 1:]).all(), "coordinate out of key range"
    return ((C[:, 0] << (3 * AXIS_BITS))
            | ((C[:, 1] + AXIS_OFF) << (2 * AXIS_BITS))
            | ((C[:, 2] + AXIS_OFF) << AXIS_BITS)
            | (C[:, 3] + AXIS_OFF))


def unique_first_occurrence(C: np.ndarray):
    """rows of C de-duplicated, in order of first occurrence.  -> (first_idx (M,), inverse (N,))."""
    keys = pack_keys(C)
    if keys.shape[0] == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    _, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(order.shape[0])
    return first[order].astype(np.int64), rank[inv.reshape(-1)].astype(np.int64)


# ----------------------------------------------------------------------------------------------
# ME.utils.batched_coordinates  (tools/diff_completion_pipeline.py:69, models/models.py:163; App. A.1)
# ----------------------------------------------------------------------------------------------
def batched_coordinates(coords_list, dtype=torch.float32) -> torch.Tensor:
    out = []
    for b, c in enumerate(coords_list):
        c = torch.as_tensor(c)
        col = torch.full((c.shape[0], 1), b, dtype=dtype)
        out.append(torch.cat([col, c.to(dtype)], dim=1))
    return torch.cat(out, dim=0)


# ----------------------------------------------------------------------------------------------
# quantisation rule of the reference: coord = torch.round(x / resolution)
#   tools/diff_completion_pipeline.py:71-72 (all four columns), utils/collations.py:8-12 (cols 1:)
# torch.round is round-half-to-even.  `div_mode`:
#   "div": true fp32 division (PyTorch CPU)            "mul": x * fp32(1/resolution)  (PyTorch's CUDA
#   scalar-divide lowering; the reference runs on CUDA) -- SURVEY.md App. B.6.
# ----------------------------------------------------------------------------------------------
def quantize(x: torch.Tensor, resolution: float, div_mode: str = "mul") -> torch.Tensor:
    x = x.to(torch.float32)
    if div_mode == "div":
        q = x / torch.tensor(resolution, dtype=torch.float32)
    elif div_mode == "mul":
        inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(resolution, dtype=torch.float32)
        q = x * inv
    else:
        raise ValueError(div_mode)
    return torch.round(q)


class TensorField:
    """ME.TensorField as used at pipeline:74-80 (App. A.2): float features + integer-valued float
    coordinates [b,x,y,z]; owns its own coordinate manager (`Geometry`)."""

    def __init__(self, features: torch.Tensor, coordinates: torch.Tensor):
        self.F = features
        self.C = coordinates
        self.geom = None  # created by sparse()

    def sparse(self) -> "SparseTensor":
        Ci = torch.floor(self.C).to(torch.int64).numpy()
        first, inv = unique_first_occurrence(Ci)
        M = first.shape[0]
        inv_t = torch.from_numpy(inv)
        sums = torch.zeros(M, self.F.shape[1], dtype=self.F.dtype)
        sums.index_add_(0, inv_t, self.F)
        cnt = torch.bincount(inv_t, minlength=M).to(self.F.dtype)
        Fv = sums / cnt[:, None]                      # UNWEIGHTED_AVERAGE
        self.geom = Geometry(Ci[first].astype(np.int32), inv)
        return SparseTensor(Fv, self.geom, 1)


class Geometry:
    """One coordinate manager: the level-0 voxel set of a TensorField plus every map derived from
    it (stride maps App. A.3, kernel maps App. A.4/A.5), cached by key exactly like ME caches them."""

    def __init__(self, C0: np.ndarray, inverse: np.ndarray):
        self.levels = {1: C0}            # tensor stride -> (M,4) int32
        self.inverse = inverse           # point -> level-0 row
        self.fine2coarse = {}            # ts_out -> (M_fine,) parent row
        self._kmaps = {}

    # -- App. A.3 -----------------------------------------------------------------------------
    def stride_level(self, ts_out: int) -> np.ndarray:
        if ts_out in self.levels:
            return self.levels[ts_out]
        Cf = self.stride_level(ts_out // 2).astype(np.int64)
        Cc = Cf.copy()
        Cc[:, 1:] = np.floor_divide(Cf[:, 1:], ts_out) * ts_out      # true floor for negatives
        first, inv = unique_first_occurrence(Cc)
        self.levels[ts_out] = Cc[first].astype(np.int32)
        self.fine2coarse[ts_out] = inv
        return self.levels[ts_out]

    # -- App. A.4 / A.5 -----------------------------------------------------------------------
    @staticmethod
    def kernel_offsets(ks: int, ts_in: int) -> np.ndarray:
        """(K,3) xyz offsets, k = kx + ks*ky + ks^2*kz (x fastest). odd ks centred, even ks not."""
        r = np.arange(ks)
        kz, ky, kx = np.meshgrid(r, r, r, indexing="ij")
        k = np.stack([kx.reshape(-1), ky.reshape(-1), kz.reshape(-1)], 1)
        if ks % 2 == 1:
            k = k - ks // 2
        return k.astype(np.int64) * ts_in

    def kernel_map(self, ts_in: int, ks: int, stride: int, transposed: bool = False):
        """list over k of (in_rows, out_rows) int64 arrays (cross-correlation convention)."""
        key = (ts_in, ks, stride, transposed)
        if key in self._kmaps:
            return self._kmaps[key]
        if transposed:
            # swap in/out of the forward stride map fine(ts_in/stride) -> coarse(ts_in)   (App. A.5)
            fwd = self.kernel_map(ts_in // stride, ks, stride, False)
            maps = [(o, i) for (i, o) in fwd]
        else:
            C_in = self.stride_level(ts_in).astype(np.int64)
            C_out = self.stride_level(ts_in * stride).astype(np.int64)
            keys_in = pack_keys(C_in)
            order = np.argsort(keys_in, kind="stable")
            sorted_keys = keys_in[order]
            maps = []
            for off in self.kernel_offsets(ks, ts_in):
                q = C_out.copy()
                q[:, 1:] += off[None, :]
                ok = in_key_range(q[:, 1:])
                qk = pack_keys(np.where(ok[:, None], q, 0))
                pos = np.searchsorted(sorted_keys, qk)
                pos = np.minimum(pos, sorted_keys.shape[0] - 1)
                hit = ok & (sorted_keys[pos] == qk)
                out_rows = np.nonzero(hit)[0]
                in_rows = order[pos[hit]]
                maps.append((in_rows.astype(np.int64), out_rows.astype(np.int64)))
        self._kmaps[key] = maps
        return maps


class SparseTensor:
    """ME.SparseTensor: `.F` (M,C) features, `.C` (M,4) int32 [b,x,y,z], tensor stride."""

    def __init__(self, F: torch.Tensor, geom: Geometry, ts: int):
        self.F, self.geom, self.ts = F, geom, ts

    @property
    def C(self) -> torch.Tensor:
        return torch.from_numpy(self.geom.stride_level(self.ts))

    def replace(self, F):
        return SparseTensor(F, self.geom, self.ts)

    def __mul__(self, w: torch.Tensor):          # minkunet.py:431  `x0*w0`
        return self.replace(self.F * w)

    def __add__(self, o: "SparseTensor"):        # minkunet.py:79
        assert o.geom is self.geom and o.ts == self.ts
        return self.replace(self.F + o.F)

    def slice(self, field: TensorField) -> torch.Tensor:     # minkunet.py:497 (App. A.6)
        assert field.geom is self.geom and self.ts == 1
        return self.F[torch.from_numpy(self.geom.inverse)]


def cat(a: SparseTensor, b: SparseTensor) -> SparseTensor:   # ME.cat, minkunet.py:464
    assert a.geom is b.geom and a.ts == b.ts
    return a.replace(torch.cat([a.F, b.F], dim=1))


# ----------------------------------------------------------------------------------------------
# MinkowskiConvolution / MinkowskiConvolutionTranspose forward  (App. A.4 / A.5)
#   out[o] = sum_k sum_{(i->o) in map_k} in[i] @ W[k]   -- per-offset gather -> GEMM -> scatter-add,
#   the algorithm of ME's CPU backend.
# ----------------------------------------------------------------------------------------------
def conv(x: SparseTensor, W: torch.Tensor, ks: int, stride: int = 1, transposed: bool = False) -> SparseTensor:
    if W.dim() == 2:                              # kernel_size=1, stride=1  (minkunet.py:72)
        assert ks == 1 and stride == 1
        return x.replace(x.F @ W.to(x.F.dtype))
    ts_out = x.ts // stride if transposed else x.ts * stride
    maps = x.geom.kernel_map(x.ts, ks, stride, transposed)
    M_out = x.geom.stride_level(ts_out).shape[0]
    W = W.to(x.F.dtype)
    out = torch.zeros(M_out, W.shape[2], dtype=x.F.dtype)
    for k, (i_rows, o_rows) in enumerate(maps):
        if i_rows.shape[0] == 0:
            continue
        out.index_add_(0, torch.from_numpy(o_rows), x.F[torch.from_numpy(i_rows)] @ W[k])
    return SparseTensor(out, x.geom, ts_out)


def batchnorm_eval(F: torch.Tensor, bn: dict, eps: float = 1e-5) -> torch.Tensor:
    """MinkowskiBatchNorm in eval mode = nn.BatchNorm1d on .F (App. A.6; pipeline:31-33)."""
    dt = F.dtype
    return ((F - bn["running_mean"].to(dt)) / torch.sqrt(bn["running_var"].to(dt) + eps)
            * bn["weight"].to(dt) + bn["bias"].to(dt))


# ----------------------------------------------------------------------------------------------
# pykeops argKmin(1) as used in MinkUNetDiff.match_part_to_full  (minkunet.py:403-418; App. A.10)
# ----------------------------------------------------------------------------------------------
def match_part_to_full(C_full: torch.Tensor, C_part: torch.Tensor, chunk: int = 8192) -> torch.Tensor:
    full_c = C_full.clone().float()
    part_c = C_part.clone().float()
    max_coord = full_c.max()
    full_c[:, 0] *= max_coord * 2.0
    part_c[:, 0] *= max_coord * 2.0
    idx = torch.empty(full_c.shape[0], dtype=torch.int64)
    for s in range(0, full_c.shape[0], chunk):
        d = ((full_c[s:s + chunk, None, :] - part_c[None, :, :]) ** 2).sum(-1)
        idx[s:s + chunk] = torch.argmin(d, dim=1)      # ties -> lowest key index
    return idx
