"""The three sparse-conv networks of LiDiff on the lidiff_b200 operator surface.

Same public classes, constructor kwargs, attribute / state-dict names and forward signatures as
/root/reference/lidiff/models/minkunet.py (MinkGlobalEnc :83-141, MinkUNetDiff :144-497,
MinkUNet :500-619; blocks :13-80), so Lightning checkpoints written by the reference load with
`load_state_dict` unchanged (SURVEY.md App. A.7).  The module tree is generated from the channel
plan instead of being spelled out stage by stage.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import me as ME
from .gate import GateMul, TakeRows
from .keops import LazyTensor

__all__ = ["MinkGlobalEnc", "MinkUNetDiff", "MinkUNet"]

_CHANNELS = (32, 32, 64, 128, 256, 256, 128, 96, 96)


def _conv_bn_relu(conv_cls, inc, outc, ks, stride, D):
    return nn.Sequential(conv_cls(inc, outc, kernel_size=ks, stride=stride, dimension=D),
                         ME.MinkowskiBatchNorm(outc), ME.MinkowskiReLU(inplace=True))


class BasicConvolutionBlock(nn.Module):
    def __init__(self, inc, outc, ks=3, stride=1, dilation=1, D=3):
        super().__init__()
        self.net = _conv_bn_relu(ME.MinkowskiConvolution, inc, outc, ks, stride, D)

    def forward(self, x):
        return self.net(x)


class BasicDeconvolutionBlock(nn.Module):
    def __init__(self, inc, outc, ks=3, stride=1, D=3):
        super().__init__()
        self.net = _conv_bn_relu(ME.MinkowskiConvolutionTranspose, inc, outc, ks, stride, D)

    def forward(self, x):
        return self.net(x)


class ResidualBlock(nn.Module):
    def __init__(self, inc, outc, ks=3, stride=1, dilation=1, D=3):
        super().__init__()
        self.net = nn.Sequential(
            ME.MinkowskiConvolution(inc, outc, kernel_size=ks, stride=stride, dimension=D),
            ME.MinkowskiBatchNorm(outc), ME.MinkowskiReLU(inplace=True),
            ME.MinkowskiConvolution(outc, outc, kernel_size=ks, stride=1, dimension=D),
            ME.MinkowskiBatchNorm(outc))
        identity = inc == outc and stride == 1
        self.downsample = nn.Sequential() if identity else nn.Sequential(
            ME.MinkowskiConvolution(inc, outc, kernel_size=1, stride=stride, dimension=D),
            ME.MinkowskiBatchNorm(outc))
        self.relu = ME.MinkowskiReLU(inplace=True)

    def forward(self, x):
        return self.relu(self.net(x) + self.downsample(x))


def _mlp(cin, hidden, cout):
    return nn.Sequential(nn.Linear(cin, hidden), nn.LeakyReLU(0.1, inplace=True), nn.Linear(hidden, cout))


class _Backbone(nn.Module):
    """stem + 4 strided encoder stages (+ 4 decoder stages) shared by all three networks."""

    def _build_encoder(self, in_channels, cs, D):
        self.stem = nn.Sequential(
            ME.MinkowskiConvolution(in_channels, cs[0], kernel_size=3, stride=1, dimension=D),
            ME.MinkowskiBatchNorm(cs[0]), ME.MinkowskiReLU(True),
            ME.MinkowskiConvolution(cs[0], cs[0], kernel_size=3, stride=1, dimension=D),
            ME.MinkowskiBatchNorm(cs[0]), ME.MinkowskiReLU(inplace=True))
        for n in range(1, 5):
            cin, cout = cs[n - 1], cs[n]
            setattr(self, f"stage{n}", nn.Sequential(
                BasicConvolutionBlock(cin, cin, ks=2, stride=2, dilation=1, D=D),
                ResidualBlock(cin, cout, ks=3, stride=1, dilation=1, D=D),
                ResidualBlock(cout, cout, ks=3, stride=1, dilation=1, D=D)))

    def _build_decoder(self, cs, D):
        for n in range(1, 5):
            cin, cout, cskip = cs[3 + n], cs[4 + n], cs[4 - n]
            setattr(self, f"up{n}", nn.ModuleList([
                BasicDeconvolutionBlock(cin, cout, ks=2, stride=2, D=D),
                nn.Sequential(ResidualBlock(cout + cskip, cout, ks=3, stride=1, dilation=1, D=D),
                              ResidualBlock(cout, cout, ks=3, stride=1, dilation=1, D=D))]))

    def weight_initialization(self):
        for m in self.modules():
            if isinstance(m, nn.BatchNorm1d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def _up(self, n, x, skip):
        up = getattr(self, f"up{n}")
        return up[1](ME.cat(up[0](x), skip))


class MinkGlobalEnc(_Backbone):
    def __init__(self, **kwargs):
        super().__init__()
        cr = kwargs.get("cr", 1.0)
        cs = [int(cr * c) for c in _CHANNELS]
        self.embed_dim = cs[-1]
        self.run_up = kwargs.get("run_up", True)
        self.D = kwargs.get("D", 3)
        self._build_encoder(kwargs.get("in_channels", 3), cs, self.D)
        self.weight_initialization()

    def forward(self, x):
        h = self.stem(x.sparse())
        for n in range(1, 5):
            h = getattr(self, f"stage{n}")(h)
        return h


class MinkUNetDiff(_Backbone):
    _GATES = ("stage1", "stage2", "stage3", "stage4", "up1", "up2", "up3", "up4")

    def __init__(self, **kwargs):
        super().__init__()
        cr = kwargs.get("cr", 1.0)
        cs = [int(cr * c) for c in _CHANNELS]
        self.embed_dim = cs[-1]
        self.run_up = kwargs.get("run_up", True)
        self.D = kwargs.get("D", 3)
        self._build_encoder(kwargs.get("in_channels", 3), cs, self.D)
        self._build_decoder(cs, self.D)
        # conditioning gates: latent (part feature), *_temp (time embedding), latemp (fusion -> channel weights)
        for g, name in enumerate(self._GATES):
            hidden = cs[4] if g < 5 else cs[g]
            setattr(self, f"latent_{name}", _mlp(cs[4], cs[4], cs[4]))
            setattr(self, f"latemp_{name}", _mlp(cs[4] + cs[4], hidden, cs[g]))
            setattr(self, f"{name}_temp", _mlp(self.embed_dim, self.embed_dim, cs[4]))
        self.last = _mlp(cs[8], 20, 3)
        self.weight_initialization()

    def get_timestep_embedding(self, timesteps):
        assert len(timesteps.shape) == 1
        half_dim = self.embed_dim // 2
        freq = np.exp(np.arange(0, half_dim) * -(np.log(10000) / (half_dim - 1)))
        freq = torch.from_numpy(freq).float().to(timesteps.device)
        arg = timesteps[:, None] * freq[None, :]
        emb = torch.cat([torch.sin(arg), torch.cos(arg)], dim=1)
        if self.embed_dim % 2 == 1:
            emb = nn.functional.pad(emb, (0, 1), "constant", 0)
        return emb

    def _match_index(self, x_full, x_part):
        """row of x_part nearest to every row of x_full, within the row's batch"""
        full_c = x_full.C.clone().float()
        part_c = x_part.C.clone().float()
        scale = full_c.max() * 2.0                       # "hash" the batch coordinate apart
        full_c[:, 0] *= scale
        part_c[:, 0] *= scale
        d = ((LazyTensor(full_c[:, None, :]) - LazyTensor(part_c[None, :, :])) ** 2).sum(-1)
        return d.argKmin(1, dim=1)[:, 0]

    def match_part_to_full(self, x_full, x_part):
        return x_part.F[self._match_index(x_full, x_part)]

    def _gate_hoisted(self, name, x, part_feats, temp_emb):
        """the gate with gradients.  The three MLPs act row by row and a voxel row's inputs are those of its part voxel and its
        batch, so they run once per part row and every voxel row gathers its result (GateMul): the same expression as _gate's,
        without saving the MLPs' activations per voxel row."""
        part_batch = part_feats.C[:, 0].long()
        absent = torch.nonzero(torch.bincount(part_batch, minlength=temp_emb.shape[0])[: temp_emb.shape[0]] == 0)[:, 0].tolist()
        if absent:
            raise ValueError(f"MinkUNetDiff: no part voxel in batch {absent}: a voxel of that batch would take another scan's condition")
        p = getattr(self, f"latent_{name}")(part_feats.F)
        t = TakeRows.apply(getattr(self, f"{name}_temp")(temp_emb), part_batch)
        pair = (t, p) if name == "up1" else (p, t)
        table = getattr(self, f"latemp_{name}")(torch.cat(pair, -1))
        return x._like(GateMul.apply(x.F, table, self._match_index(x, part_feats)))

    def _gate(self, g, x, part_feats, temp_emb):
        name = self._GATES[g]
        mlps = [getattr(self, f"latent_{name}"), getattr(self, f"{name}_temp"), getattr(self, f"latemp_{name}")]
        if torch.is_grad_enabled() and (x.F.requires_grad or part_feats.F.requires_grad or temp_emb.requires_grad
                                        or any(w.requires_grad for m in mlps for w in m.parameters())):
            return self._gate_hoisted(name, x, part_feats, temp_emb)
        p = mlps[0](self.match_part_to_full(x, part_feats))
        t = mlps[1](temp_emb)
        per_batch = torch.unique(x.C[:, 0], return_counts=True)[1]
        t = torch.repeat_interleave(t, per_batch, dim=0)
        pair = (t, p) if name == "up1" else (p, t)       # the reference concatenates (t4, p4) for up1 only
        return x * mlps[2](torch.cat(pair, -1))

    def forward(self, x, x_sparse, part_feats, t):
        temp_emb = self.get_timestep_embedding(t)
        skips = [self.stem(x_sparse)]
        for n in range(1, 5):
            skips.append(getattr(self, f"stage{n}")(self._gate(n - 1, skips[-1], part_feats, temp_emb)))
        y = skips[4]
        for n in range(1, 5):
            y = self._up(n, self._gate(3 + n, y, part_feats, temp_emb), skips[4 - n])
        return self.last(y.slice(x).F)


class MinkUNet(_Backbone):
    def __init__(self, **kwargs):
        super().__init__()
        cr = kwargs.get("cr", 1.0)
        cs = [int(cr * c) for c in _CHANNELS]
        self.run_up = kwargs.get("run_up", True)
        self.D = kwargs.get("D", 3)
        self._build_encoder(kwargs.get("in_channels", 3), cs, self.D)
        self._build_decoder(cs, self.D)
        self.last = nn.Sequential(nn.Linear(cs[8], 20), nn.LeakyReLU(0.1, inplace=True),
                                  nn.Linear(20, kwargs.get("out_channels", 3)), nn.Tanh())
        self.weight_initialization()
        self.dropout = nn.Dropout(0.3, True)

    def forward(self, x):
        skips = [self.stem(x.sparse())]
        for n in range(1, 5):
            skips.append(getattr(self, f"stage{n}")(skips[-1]))
        y = skips[4]
        for n in range(1, 5):
            y = self._up(n, y, skips[4 - n])
        return self.last(y.slice(x).F)
