"""Per-layer timing of the sparse convolution variants (FFMA vs wgmma) on the real 180k-point
geometry (development aid).  Usage: python scripts/bench_layers.py [sigma]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lidiff_b200 import _lib                                   # noqa: E402
from lidiff_b200._lib import ConvDesc, ConvIO                  # noqa: E402
from lidiff_b200.engine import Geometry                        # noqa: E402
from lidiff_b200.preprocess import farthest_point_sample       # noqa: E402
from lidiff_b200.synth import range_filter, synthetic_scan     # noqa: E402

LAYERS = [  # level, c1, c2, cout, kind
    (0, 32, 0, 32, "3"), (0, 96, 32, 96, "3"), (0, 96, 0, 96, "3"),
    (1, 32, 0, 32, "3"), (1, 96, 32, 96, "3"), (1, 32, 0, 32, "dn"),
    (2, 64, 0, 64, "3"), (2, 128, 64, 128, "3"), (2, 128, 0, 128, "3"),
    (3, 128, 0, 128, "3"), (3, 256, 128, 256, "3"), (3, 256, 0, 256, "3"), (3, 256, 0, 256, "up"), (3, 256, 128, 256, "1"),
    (4, 256, 0, 256, "3"), (4, 128, 0, 128, "dn"),
]


def main():
    sigma = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    dev = "cuda:0"
    h = _lib.get_handle(dev)
    raw = torch.tensor(range_filter(synthetic_scan(0)), device=dev)
    scan = raw[farthest_point_sample(raw, 18000)].repeat(10, 1)
    N = scan.shape[0]
    g = torch.Generator(device=dev).manual_seed(0)
    x = (scan + sigma * torch.randn(scan.shape, device=dev, generator=g, dtype=torch.float64)).float()
    coords = torch.zeros(N, 4, device=dev)
    coords[:, 1:] = torch.round(x * 20.0)
    geo = Geometry(h, N)
    geo.build(coords, N)
    sizes = geo.sizes()
    print(f"sigma={sigma} level sizes {sizes}")
    for l in range(5):
        nb = geo.nbr3[l][:, :sizes[l]]
        print(f"  L{l}: pairs {(nb >= 0).sum().item()}  avg nbrs {(nb >= 0).sum().item() / max(sizes[l], 1):.2f}")
    print(f"{'layer':34s} {'pairs':>9s} {'GF(2p)':>8s} {'ffma ms':>8s} {'tc ms':>8s} {'tc+perm':>8s} {'TF/s useful':>12s} {'TF/s dense-eq':>14s}")
    for (lvl, c1, c2, cout, kind) in LAYERS:
        if kind == "3":
            nbr, kvol, M, perm = geo.nbr3[lvl], 27, sizes[lvl], geo.perm3[lvl]
        elif kind == "dn":
            nbr, kvol, M, perm = geo.nbr_dn[lvl], 8, sizes[lvl], geo.perm_dn[lvl]
        elif kind == "up":
            nbr, kvol, M, perm = geo.nbr_up[lvl], 8, sizes[lvl], geo.perm_up[lvl]
        else:
            nbr, kvol, M, perm = None, 1, sizes[lvl], None
        pairs = int((nbr[:, :M] >= 0).sum().item()) if nbr is not None else M
        W = torch.randn(kvol, c1 + c2, cout, device=dev) * 0.05
        Wp = h.pack_weights(W)
        a = torch.randn(2, N, c1, device=dev)
        b = torch.randn(2, N, c2, device=dev) if c2 else None
        out = torch.empty(2, N, cout, device=dev)
        sc, sh = torch.rand(cout, device=dev) + 0.5, torch.randn(cout, device=dev)
        d = ConvDesc()
        d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, kvol
        d.weight, d.weight_packed = W.data_ptr(), (Wp.data_ptr() if Wp is not None else None)
        d.scale, d.shift, d.relu = sc.data_ptr(), sh.data_ptr(), 1
        d.nbr = nbr.data_ptr() if nbr is not None else None
        d.nbr_stride = N
        d.d_mout, d.mout_cap, d.npass = geo.d_n[lvl].data_ptr(), N, 2
        for p in range(2):
            d.io[p] = ConvIO(a[p].data_ptr(), b[p].data_ptr() if b is not None else None, None, out[p].data_ptr(), None, None, None)
        res = {}
        for algo in (1, 2, 3):
            d.row_perm = perm.data_ptr() if (algo == 3 and perm is not None) else None
            algo_ = 2 if algo == 3 else algo
            if algo_ == 2 and Wp is None:
                res[algo] = float("nan")
                continue
            for _ in range(2):
                h.spconv(d, algo_)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                h.spconv(d, algo_)
            e1.record()
            torch.cuda.synchronize()
            res[algo] = e0.elapsed_time(e1) / 5
            if algo == 1:
                ref = out.clone()
            elif algo == 2:
                err = ((out[:, :M] - ref[:, :M]).abs().max() / ref[:, :M].abs().max()).item()
        gf = 2 * 2.0 * pairs * (c1 + c2) * cout / 1e9
        dense = 2 * 2.0 * M * kvol * (c1 + c2) * cout / 1e9
        name = f"L{lvl} {c1}+{c2}->{cout} k{kvol} {kind}"
        tcms = res[2]
        print(f"{name:34s} {pairs:9d} {gf:8.1f} {res[1]:8.3f} {tcms:8.3f} {res[3]:8.3f} {gf / res[3]:12.1f} {dense / tcms:14.1f}   maxrel {err:.1e}")


if __name__ == "__main__":
    main()
