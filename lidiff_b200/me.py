"""MinkowskiEngine operator surface, H100-native underneath.

Mirrors exactly the subset of `import MinkowskiEngine as ME` that the reference hot path uses
(SURVEY.md 8b; call sites /root/reference/lidiff/models/minkunet.py:17-24,36-42,53-76,94-99,464,497
and /root/reference/lidiff/tools/diff_completion_pipeline.py:69-80,149): same names, argument
meaning, attribute names (`.F`, `.C`, `.kernel`, `.bn`) and error behaviour (RuntimeError).
Every operator is one call into the C-ABI CUDA library (`lidiff_b200._lib`); torch supplies device
memory and streams only.  There is no CPU implementation: CPU tensors raise.

This is the generic (operator-by-operator) path; `lidiff_b200.engine` runs the same kernels fused
and sync-free for the sampling loop.
"""
from __future__ import annotations

import math
from enum import Enum

import torch
import torch.nn as nn

from . import _lib
from ._lib import ConvDesc, ConvIO


class SparseTensorQuantizationMode(Enum):
    RANDOM_SUBSAMPLE = 0
    UNWEIGHTED_AVERAGE = 1
    UNWEIGHTED_SUM = 2
    NO_QUANTIZATION = 3


class MinkowskiAlgorithm(Enum):
    DEFAULT = 0
    MEMORY_EFFICIENT = 1
    SPEED_OPTIMIZED = 2


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f"lidiff_b200.me: {what} must live on a CUDA device (no CPU backend)")


class _Level:
    """coordinates of one tensor stride + its hash grid"""
    __slots__ = ("C", "n", "d_n", "grid", "parent_inverse")

    def __init__(self, C, n, d_n, grid, parent_inverse=None):
        self.C, self.n, self.d_n, self.grid, self.parent_inverse = C, n, d_n, grid, parent_inverse


class CoordinateManager:
    """Per-TensorField coordinate manager: level-0 voxel set, strided levels, kernel maps (cached by
    key like ME's manager; SURVEY.md App. A.2-A.5)."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.h = _lib.get_handle(self.device)
        self.levels = {}
        self.kmaps = {}
        self.field_inverse = None

    def _unique(self, in_f, in_i, n_in, ts_floor):
        h, dev = self.h, self.device
        grid = h.new_grid(n_in)
        out = torch.empty((n_in, 4), dtype=torch.int32, device=dev)
        inv = torch.empty(n_in, dtype=torch.int32, device=dev)
        d_n = torch.zeros(1, dtype=torch.int32, device=dev)
        h.unique_build(in_f, in_i, None, n_in, ts_floor, grid, out, inv, d_n, h.unique_scratch(n_in))
        n = int(d_n.item())
        # only the level-0 insertion can leave the key range (coarser levels floor coordinates that are already in range): one status
        # read per TensorField, right behind the build that could have raised it (the word is per device and cleared by the read)
        if ts_floor == 0 and (h.read_status() & 1):
            raise RuntimeError("lidiff_b200.me: coordinate outside the supported key range "
                               "(-131072 <= x <= 131071 voxels, 0 <= batch < 1024, no NaN)")
        return _Level(out[:n], n, d_n, grid, inv)

    def insert_field(self, coords_f: torch.Tensor):
        lvl = self._unique(coords_f.contiguous(), None, coords_f.shape[0], 0)
        self.levels[1] = lvl
        self.field_inverse = lvl.parent_inverse
        return lvl

    def level(self, ts: int) -> _Level:
        if ts not in self.levels:
            parent = self.level(ts // 2)
            self.levels[ts] = self._unique(None, parent.C.contiguous(), parent.n, ts)
        return self.levels[ts]

    def kernel_map(self, ts_in: int, ks: int, stride: int, transposed: bool) -> torch.Tensor:
        key = (ts_in, ks, stride, transposed)
        if key not in self.kmaps:
            if transposed:
                lin, lout, step = self.level(ts_in), self.level(ts_in // stride), -(ts_in // stride)
            else:
                lin, lout, step = self.level(ts_in), self.level(ts_in * stride), ts_in
            nbr = torch.empty((ks ** 3, lout.n), dtype=torch.int32, device=self.device)
            self.h.kernel_map(lin.grid, lout.C, None, lout.n, ks, step, nbr, lout.n)
            self.kmaps[key] = nbr
        return self.kmaps[key]


class TensorField:
    """ME.TensorField(features, coordinates, quantization_mode, minkowski_algorithm, device)"""

    def __init__(self, features, coordinates, quantization_mode=SparseTensorQuantizationMode.UNWEIGHTED_AVERAGE,
                 minkowski_algorithm=MinkowskiAlgorithm.DEFAULT, device=None, coordinate_manager=None, **_):
        if device is not None:
            features, coordinates = features.to(device), coordinates.to(device)
        _require_cuda(features, "TensorField features")
        if quantization_mode != SparseTensorQuantizationMode.UNWEIGHTED_AVERAGE:
            raise RuntimeError("lidiff_b200.me: only UNWEIGHTED_AVERAGE quantisation is implemented (the mode the reference uses)")
        if coordinates.shape[0] != features.shape[0] or coordinates.shape[1] != 4:
            raise RuntimeError("TensorField: coordinates must be (N,4) [b,x,y,z] matching features rows")
        self._F = features.float().contiguous()
        self._C = coordinates.float().contiguous()
        self.coordinate_manager = coordinate_manager or CoordinateManager(features.device)
        self._sparse = None

    F = property(lambda self: self._F)
    C = property(lambda self: self._C)
    features = F
    coordinates = C
    device = property(lambda self: self._F.device)

    @property
    def inverse_mapping(self):
        if self.coordinate_manager.field_inverse is None:
            self.sparse()
        return self.coordinate_manager.field_inverse.long()

    def sparse(self, tensor_stride=1, **_):
        if tensor_stride != 1:
            raise RuntimeError("TensorField.sparse: only tensor_stride=1 is implemented")
        cm = self.coordinate_manager
        if 1 not in cm.levels:
            cm.insert_field(self._C)
        if torch.is_grad_enabled() and self._F.requires_grad:
            out = _VoxelMean.apply(self._F, cm)
        else:
            out = _voxel_mean(self._F, cm)
        return SparseTensor(out, coordinate_manager=cm, tensor_stride=1)


def _voxel_mean(F, cm):
    lvl = cm.levels[1]
    n, c = F.shape
    out = torch.empty((lvl.n, c), dtype=torch.float32, device=F.device)
    cm.h.voxel_mean(F, cm.field_inverse, n, c, None, lvl.n, out, cm.h.voxel_mean_scratch(lvl.n, c))
    return out


def _gather(src, cm, n):
    out = torch.empty((n, src.shape[1]), dtype=torch.float32, device=src.device)
    cm.h.gather_rows(src, cm.field_inverse, n, src.shape[1], out)
    return out


class _VoxelMean(torch.autograd.Function):
    """TensorField.sparse(): the mean of each voxel's points; backward: every point gets its voxel's gradient / member count"""

    @staticmethod
    def forward(ctx, F, cm):
        ctx.cm, ctx.n = cm, F.shape[0]
        return _voxel_mean(F, cm)

    @staticmethod
    def backward(ctx, grad):
        cm = ctx.cm
        count = torch.bincount(cm.field_inverse.long(), minlength=grad.shape[0]).to(grad.dtype)
        return _gather((grad / count[:, None]).contiguous(), cm, ctx.n), None


class _Slice(torch.autograd.Function):
    """SparseTensor.slice(): every point takes its voxel's row; backward: per voxel, the sum of its points' gradients in point
    order (rowsum.index_sum: no atomics, the same bits on every run)"""

    @staticmethod
    def forward(ctx, F, cm, n):
        ctx.cm = cm
        return _gather(F, cm, n)

    @staticmethod
    def backward(ctx, grad):
        from .rowsum import index_sum
        cm = ctx.cm
        return index_sum(grad.float(), cm.field_inverse, cm.levels[1].n), None, None


class SparseTensor:
    """ME.SparseTensor: `.F` (M,C) fp32, `.C` (M,4) int32 [b,x,y,z]."""

    def __init__(self, features, coordinates=None, coordinate_manager=None, tensor_stride=1, device=None, **_):
        if coordinate_manager is None:
            if coordinates is None:
                raise RuntimeError("SparseTensor needs coordinates or a coordinate_manager")
            if device is not None:
                features, coordinates = features.to(device), coordinates.to(device)
            # ME.SparseTensor(features=, coordinates=): quantise with the default RANDOM_SUBSAMPLE ->
            # here: keep the first occurrence of each coordinate
            cm = CoordinateManager(features.device)
            lvl = cm.insert_field(coordinates.float())
            first = torch.full((lvl.n,), features.shape[0], dtype=torch.long, device=features.device)
            first.scatter_reduce_(0, cm.field_inverse.long(), torch.arange(features.shape[0], device=features.device), "amin")
            features = features[first]
            coordinate_manager = cm
        _require_cuda(features, "SparseTensor features")
        self._F = features
        self.coordinate_manager = coordinate_manager
        self.tensor_stride = tensor_stride if isinstance(tensor_stride, int) else int(tensor_stride[0])

    F = property(lambda self: self._F)
    features = F
    device = property(lambda self: self._F.device)

    @property
    def C(self):
        return self.coordinate_manager.level(self.tensor_stride).C

    coordinates = C

    def _like(self, F):
        return SparseTensor(F, coordinate_manager=self.coordinate_manager, tensor_stride=self.tensor_stride)

    def _same_map(self, o):
        if o.coordinate_manager is not self.coordinate_manager or o.tensor_stride != self.tensor_stride:
            raise RuntimeError("SparseTensor arithmetic needs operands on the same coordinate map")

    def __mul__(self, o):
        if isinstance(o, SparseTensor):
            self._same_map(o)
            o = o.F
        return self._like(self._F * o)

    def __add__(self, o):
        if isinstance(o, SparseTensor):
            self._same_map(o)
            o = o.F
        return self._like(self._F + o)

    def slice(self, field: TensorField) -> TensorField:
        if field.coordinate_manager is not self.coordinate_manager or self.tensor_stride != 1:
            raise RuntimeError("slice: tensor field and sparse tensor must share the stride-1 coordinate map")
        cm = self.coordinate_manager
        n = field.F.shape[0]
        if torch.is_grad_enabled() and self._F.requires_grad:
            out = _Slice.apply(self._F.contiguous(), cm, n)
        else:
            out = _gather(self._F.contiguous(), cm, n)
        return TensorField(out, field.C, coordinate_manager=cm)


def cat(*tensors):
    a = tensors[0]
    for t in tensors[1:]:
        a._same_map(t)
    return a._like(torch.cat([t.F for t in tensors], dim=1))


# ---------------------------------------------------------------------------------------------------
# layers
# ---------------------------------------------------------------------------------------------------
class _ConvBase(nn.Module):
    transposed = False

    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, bias=False,
                 kernel_generator=None, expand_coordinates=False, convolution_mode=None, dimension=None):
        super().__init__()
        if dimension != 3:
            raise RuntimeError("lidiff_b200.me: only dimension=3 is implemented")
        if dilation != 1 or bias or expand_coordinates:
            raise RuntimeError("lidiff_b200.me: dilation != 1, bias and expand_coordinates are not implemented "
                               "(the reference never uses them)")
        if kernel_size not in (1, 2, 3) or stride not in (1, 2):
            raise RuntimeError("lidiff_b200.me: kernel_size in {1,2,3} and stride in {1,2} only")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.dimension = kernel_size, stride, dimension
        self.kernel_volume = kernel_size ** 3
        if self.kernel_volume == 1 and stride == 1:
            shape = (in_channels, out_channels)                # ME stores the 1x1 kernel as a matrix
        else:
            shape = (self.kernel_volume, in_channels, out_channels)
        self.kernel = nn.Parameter(torch.empty(shape, dtype=torch.float32))
        self.bias = None
        self.reset_parameters()

    def reset_parameters(self):
        with torch.no_grad():
            n = (self.out_channels if self.transposed else self.in_channels) * self.kernel_volume
            stdv = 1.0 / math.sqrt(n)
            # not through .data: that write would leave the parameter's version, and with it the packed-weight caches, unchanged
            self.kernel.uniform_(-stdv, stdv)

    def _packed_weight(self, h):
        """tensor-core image of the kernel (fp16 hi/lo, wgmma layout), cached until the parameter changes"""
        if getattr(self, "algo", _lib.ALGO_AUTO) == _lib.ALGO_FFMA:
            return None
        W = self.kernel
        key = (W.data_ptr(), W._version)
        if getattr(self, "_pack_key", None) != key:
            W3 = W.detach() if W.dim() == 3 else W.detach()[None]
            self._pack = h.pack_weights(W3.contiguous())
            self._pack_key = key
        return self._pack.data_ptr() if self._pack is not None else None

    def forward(self, x: SparseTensor) -> SparseTensor:
        if not isinstance(x, SparseTensor):
            raise RuntimeError(f"{type(self).__name__} expects a SparseTensor")
        cm, ts = x.coordinate_manager, x.tensor_stride
        F = x.F.contiguous()
        if F.shape[1] != self.in_channels:
            raise RuntimeError(f"channel mismatch: input has {F.shape[1]}, layer expects {self.in_channels}")
        if self.transposed:
            if ts % self.stride:
                raise RuntimeError("transposed convolution below tensor stride 1")
            ts_out = ts // self.stride
        else:
            ts_out = ts * self.stride
        if torch.is_grad_enabled() and (F.requires_grad or self.kernel.requires_grad):
            out = _ConvFn.apply(F, self.kernel, self, cm, ts, ts_out)
        else:
            out = self._conv(F, cm, ts, ts_out)
        return SparseTensor(out, coordinate_manager=cm, tensor_stride=ts_out)

    def _map(self, cm, ts):
        """the forward kernel map (kvol, rows out), or None for the 1x1 identity"""
        if self.kernel.dim() == 3 and not (self.kernel_volume == 1):
            return cm.kernel_map(ts, self.kernel_size, self.stride, self.transposed)
        return None

    def _conv(self, F, cm, ts, ts_out):
        lout = cm.level(ts_out)
        W = self.kernel
        nbr = self._map(cm, ts)
        out = torch.empty((lout.n, self.out_channels), dtype=torch.float32, device=F.device)
        d = ConvDesc()
        d.c1, d.c2, d.cout, d.kvol = self.in_channels, 0, self.out_channels, self.kernel_volume
        d.weight = W.data_ptr()
        d.weight_packed = self._packed_weight(cm.h)
        d.relu = 0
        d.nbr = nbr.data_ptr() if nbr is not None else None
        d.nbr_stride = lout.n
        d.mout_cap, d.npass = lout.n, 1
        d.io[0] = ConvIO(F.data_ptr(), None, None, out.data_ptr(), None, None, None)
        if lout.n > 0:
            cm.h.spconv(d, getattr(self, "algo", _lib.ALGO_AUTO))
        return out

    # ---- backward ------------------------------------------------------------------------------------------------------------
    def _adjoint(self, cm, ts, ts_out):
        """(map, weight transform) of the input gradient: dX = conv(G) on the adjoint map with the transformed kernel.
        3x3x3 stride 1: the same map, offset k <- 26 - k (the map is symmetric: nbr[k][o] = i <=> nbr[26 - k][i] = o), W[26 - k]^T.
        k2 s2 (fine -> coarse): the transposed map coarse -> fine, W[k]^T; a transposed convolution: the strided map, W[k]^T.
        1x1: the identity, W^T."""
        W = self.kernel.detach()
        if W.dim() == 2:
            return None, W.t()[None]
        if self.kernel_volume == 1:
            return None, W.transpose(1, 2)
        if self.kernel_size == 3 and self.stride == 1:
            return cm.kernel_map(ts, 3, 1, False), W.flip(0).transpose(1, 2)
        if self.transposed:
            return cm.kernel_map(ts_out, self.kernel_size, self.stride, False), W.transpose(1, 2)
        return cm.kernel_map(ts_out, self.kernel_size, self.stride, True), W.transpose(1, 2)

    def _adjoint_packs(self, h, Wt):
        """transformed kernel slices of at most 256 (or 128) output channels, packed for the tensor cores and cached until the
        parameter changes (an optimizer step bumps its version): [(c0, c1, weight, packed)]"""
        W = self.kernel
        key = (W.data_ptr(), W._version)
        if getattr(self, "_adj_key", None) != key:
            cin = Wt.shape[2]
            # the forward kernel takes Cout <= 128 or exactly 256: 384 runs as 256 + 128, 192 as 128 + 64
            cuts = {384: (0, 256, 384), 192: (0, 128, 192)}.get(cin, (0, cin))
            packs = []
            for c0, c1 in zip(cuts[:-1], cuts[1:]):
                w = Wt[:, :, c0:c1].contiguous()
                pk = h.pack_weights(w)
                if pk is None:
                    raise RuntimeError(f"{type(self).__name__}({self.in_channels}, {self.out_channels}): no tensor-core kernel for the "
                                       f"input gradient's {c1 - c0} output channels")
                packs.append((c0, c1, w, pk))
            self._adj, self._adj_key = packs, key
        return self._adj

    def _input_grad(self, G, cm, ts, ts_out):
        nbr, Wt = self._adjoint(cm, ts, ts_out)
        lin = cm.level(ts)
        # the output gradient is the activation operand of the FP16x3 product, whose split has an absolute floor of 2^-25: scale it
        # by a power of two so that its largest magnitude lies in [8192, 16384), as the packed weights are (exact both ways).  Only
        # finite elements count, as in k_weight_absmax: a NaN or inf row makes the rows that read it non-finite whatever the scale,
        # and must not leave the others unscaled
        Ga = G.abs()
        amax = torch.where(torch.isfinite(Ga), Ga, torch.zeros_like(Ga)).amax()
        e = torch.frexp(amax).exponent
        scale = torch.where(torch.isfinite(amax) & (amax > 0), torch.ldexp(torch.ones_like(amax), (14 - e).clamp(max=126)),
                            torch.ones_like(amax))
        Gs = (G * scale).contiguous()
        parts = []
        for c0, c1, w, pk in self._adjoint_packs(cm.h, Wt):
            out = torch.empty((lin.n, c1 - c0), dtype=torch.float32, device=G.device)
            d = ConvDesc()
            d.c1, d.c2, d.cout, d.kvol = self.out_channels, 0, c1 - c0, w.shape[0]
            d.weight, d.weight_packed = w.data_ptr(), pk.data_ptr()
            d.relu = 0
            d.nbr = nbr.data_ptr() if nbr is not None else None
            d.nbr_stride = lin.n
            d.mout_cap, d.npass = lin.n, 1
            d.io[0] = ConvIO(Gs.data_ptr(), None, None, out.data_ptr(), None, None, None)
            if lin.n > 0:
                cm.h.spconv(d, _lib.ALGO_TC)
            parts.append(out)
        out = parts[0] if len(parts) == 1 else torch.cat(parts, 1)
        return out / scale

    def _weight_grad(self, F, G, cm, ts):
        nbr = self._map(cm, ts)
        dw = torch.empty((self.kernel_volume, self.in_channels, self.out_channels), dtype=torch.float32, device=G.device)
        cm.h.spconv_wgrad(F, G, nbr, self.kernel_volume, dw)
        return dw.reshape(self.kernel.shape)


class _ConvFn(torch.autograd.Function):
    """a sparse convolution with its gradients: dX on the adjoint map (the forward kernels, _ConvBase._input_grad), dW from
    lb2_spconv_wgrad.  The forward is the no-grad call itself, so its values are the same bits."""

    @staticmethod
    def forward(ctx, F, W, layer, cm, ts, ts_out):
        ctx.save_for_backward(F)
        ctx.layer, ctx.cm, ctx.ts, ctx.ts_out = layer, cm, ts, ts_out
        return layer._conv(F, cm, ts, ts_out)

    @staticmethod
    def backward(ctx, G):
        (F,) = ctx.saved_tensors
        layer, cm = ctx.layer, ctx.cm
        G = G.contiguous()
        dF = layer._input_grad(G, cm, ctx.ts, ctx.ts_out) if ctx.needs_input_grad[0] else None
        dW = layer._weight_grad(F, G, cm, ctx.ts) if ctx.needs_input_grad[1] else None
        return dF, dW, None, None, None, None


class MinkowskiConvolution(_ConvBase):
    """ME.MinkowskiConvolution(inc, outc, kernel_size=, stride=, dilation=, dimension=3)"""
    transposed = False


class MinkowskiConvolutionTranspose(_ConvBase):
    """ME.MinkowskiConvolutionTranspose(inc, outc, kernel_size=2, stride=2, dimension=3); the output
    lands on the existing finer coordinate map (SURVEY.md App. A.5)."""
    transposed = True


class MinkowskiBatchNorm(nn.Module):
    """holds `.bn = nn.BatchNorm1d` so state-dict keys (`...bn.weight`) and the reference's
    `isinstance(m, nn.BatchNorm1d)` initialisation (minkunet.py:128-132) keep working."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                                 track_running_stats=track_running_stats)

    def forward(self, x: SparseTensor) -> SparseTensor:
        return x._like(self.bn(x.F))


_SYNC_GROUPS = {}


def _sync_group(process_group):
    """the process group the sync-BN collectives run on: the given one, or else one of their own over every rank, created once per
    default group (all ranks reach their first sync-BN forward together, so they create it in the same order).  On a group of
    their own the layers' collectives cannot interleave differently from DDP's gradient all-reduces on different ranks."""
    import torch.distributed as dist
    if process_group is not None:
        return process_group
    world = dist.group.WORLD
    got = _SYNC_GROUPS.get(id(world))
    if got is None or got[0] is not world:
        got = (world, dist.new_group(ranks=list(range(dist.get_world_size()))))
        _SYNC_GROUPS[id(world)] = got
    return got[1]


class _SyncBatchNormFn(torch.autograd.Function):
    """training-mode batch norm over the rows of every rank of `group` (lb2_sync_bn_*: three collectives forward, two backward, on
    the current stream).  The parameter gradients are this rank's sums, as torch's SyncBatchNorm returns them; DDP averages them."""

    @staticmethod
    def forward(ctx, x, weight, bias, bn, group, factor):
        import torch.distributed as dist
        h = _lib.get_handle(x.device)
        n, c = x.shape
        i64 = dict(dtype=torch.int64, device=x.device)
        mw = torch.empty(2 * c, **i64)
        h.sync_bn_max(x, mw)
        dist.all_reduce(mw, dist.ReduceOp.MAX, group=group)
        sw = torch.empty(2 * c + 1, **i64)
        h.sync_bn_sum(x, mw, sw)
        dist.all_reduce(sw, group=group)
        mean = torch.empty(c, dtype=torch.float64, device=x.device)
        qw = torch.empty(4 * c, **i64)
        h.sync_bn_sumsq(x, mw, sw, mean, qw)
        dist.all_reduce(qw, group=group)
        var, invstd, y = torch.empty_like(mean), torch.empty_like(mean), torch.empty_like(x)
        track = bn.track_running_stats and bn.running_mean is not None
        h.sync_bn_apply(x, mw, sw, mean, qw, weight, bias, bn.eps, factor, bn.running_mean if track else None,
                        bn.running_var if track else None, var, invstd, y)
        ctx.save_for_backward(x, weight, mean, invstd, sw)
        ctx.group = group
        return y

    @staticmethod
    def backward(ctx, dy):
        import torch.distributed as dist
        x, weight, mean, invstd, sw = ctx.saved_tensors
        h = _lib.get_handle(x.device)
        dy = dy.contiguous()
        c = x.shape[1]
        mw = torch.empty(3 * c, dtype=torch.int64, device=x.device)
        h.sync_bn_backward_max(dy, x, mean, invstd, mw)
        dist.all_reduce(mw, dist.ReduceOp.MAX, group=ctx.group)
        bw = torch.empty(4 * c, dtype=torch.int64, device=x.device)
        dgamma = torch.empty(c, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[1] else None
        dbeta = torch.empty(c, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[2] else None
        h.sync_bn_backward_sum(dy, x, mean, invstd, mw, bw, dgamma, dbeta)
        dist.all_reduce(bw, group=ctx.group)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            h.sync_bn_backward_apply(dy, x, mean, invstd, weight, mw, bw, sw[2 * c:], dx)
        return dx, dgamma, dbeta, None, None, None


class MinkowskiSyncBatchNorm(MinkowskiBatchNorm):
    """ME.MinkowskiSyncBatchNorm: the same `.bn` (parameters, buffers, state-dict keys) as MinkowskiBatchNorm.  In training mode
    with a process group of more than one rank the statistics are those of every rank's rows (lb2_sync_bn_*: every output depends
    only on the multiset of rows, whatever their split across ranks); otherwise it is exactly MinkowskiBatchNorm, as torch's
    SyncBatchNorm falls back to BatchNorm."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, process_group=None):
        super().__init__(num_features, eps=eps, momentum=momentum, affine=affine, track_running_stats=track_running_stats)
        self.process_group = process_group

    def _world(self):
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            return 1
        return dist.get_world_size(self.process_group)

    def forward(self, x: SparseTensor) -> SparseTensor:
        if not self.training or self._world() < 2:
            return super().forward(x)
        bn = self.bn
        # the momentum and num_batches_tracked bookkeeping of nn.BatchNorm1d.forward
        factor = 0.0 if bn.momentum is None else bn.momentum
        if bn.track_running_stats and bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
            factor = 1.0 / float(bn.num_batches_tracked) if bn.momentum is None else bn.momentum
        F = x.F
        if F.dim() != 2 or F.dtype != torch.float32 or F.shape[1] != bn.num_features:
            raise RuntimeError(f"MinkowskiSyncBatchNorm({bn.num_features}): features must be (rows, {bn.num_features}) fp32")
        y = _SyncBatchNormFn.apply(F.contiguous(), bn.weight, bn.bias, bn, _sync_group(self.process_group), factor)
        return x._like(y)

    @classmethod
    def convert_sync_batchnorm(cls, module, process_group=None):
        """every MinkowskiBatchNorm in `module` replaced by a MinkowskiSyncBatchNorm holding the same `.bn` (so the same parameters,
        buffers and state-dict keys); returns the converted module, as torch.nn.SyncBatchNorm.convert_sync_batchnorm does"""
        out = module
        if isinstance(module, MinkowskiBatchNorm) and not isinstance(module, MinkowskiSyncBatchNorm):
            b = module.bn
            out = cls(b.num_features, eps=b.eps, momentum=b.momentum, affine=b.affine, track_running_stats=b.track_running_stats,
                      process_group=process_group)
            out.bn = b
            out.train(module.training)
        for name, child in module.named_children():
            out.add_module(name, cls.convert_sync_batchnorm(child, process_group))
        return out


class MinkowskiReLU(nn.Module):
    def __init__(self, inplace=False):
        super().__init__()

    def forward(self, x: SparseTensor) -> SparseTensor:
        return x._like(torch.relu(x.F))


class _Utils:
    @staticmethod
    def batched_coordinates(coords, dtype=torch.int32, device=None):
        """ME.utils.batched_coordinates: (sum N_i, D+1), column 0 = list index (SURVEY.md App. A.1)."""
        out = []
        for b, c in enumerate(coords):
            c = torch.as_tensor(c)
            if dtype in (torch.int32, torch.int64) and c.is_floating_point():
                c = torch.floor(c)
            c = c.to(dtype)
            col = torch.full((c.shape[0], 1), b, dtype=dtype, device=c.device)
            out.append(torch.cat([col, c], dim=1))
        res = torch.cat(out, dim=0)
        return res.to(device) if device is not None else res

    @staticmethod
    def sparse_quantize(coordinates, features=None, return_index=False, quantization_size=None, **_):
        """first-occurrence de-duplication of integer coordinates (lidiff/map_from_scans.py:91)."""
        c = torch.as_tensor(coordinates)
        if quantization_size is not None:
            c = torch.floor(c / quantization_size)
        c = c.to(torch.int64)
        uniq, inv = torch.unique(c, dim=0, return_inverse=True)
        first = torch.full((uniq.shape[0],), c.shape[0], dtype=torch.long)
        first.scatter_reduce_(0, inv, torch.arange(c.shape[0]), "amin")
        first = torch.sort(first).values
        if return_index:
            return c[first].int(), first
        if features is not None:
            return c[first].int(), torch.as_tensor(features)[first]
        return c[first].int()


utils = _Utils()
