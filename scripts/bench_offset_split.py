"""Times the offset split of the 3^3 tensor-core convolutions (lidiff_b200/engine.py OFFSET_RANGES, DESIGN.md §3) per layer shape.

On the benchmark scan's geometry (tests/golden/step_synth180k.npz: `part` x 10 plus sigma-noise, quantised at 5 cm) at three
schedule positions (sigma = 1.0, 0.2, 0.05), every split-eligible conv shape of the diffusion U-Net (one kernel offset per
accumulation group: stage 4 at level 4, up1 at level 3, up2's first conv at level 2; two guidance passes) runs at G = 1, 2 and 3,
alternated, each timed with CUDA events over many launches.  Prints one line per (sigma, layer, G): the median time per conv and
the MMA rows it issues (sum over its launches of 128 x popcount of each dispatched tile's offset union, counted on the host from
the row and tile orders; x passes x channel halves is the same factor for every G).

    python scripts/bench_offset_split.py [--reps 5] [--iters 20] [--out results/offset_split.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lidiff_b200 import _lib  # noqa: E402
from lidiff_b200._lib import ConvDesc, ConvIO  # noqa: E402
from lidiff_b200.engine import OFFSET_RANGES, Geometry  # noqa: E402

DEV = "cuda:0"
# (name, c1, c2, cout, level): the split-eligible 3^3 convs of MinkUNetDiff (cs = 32 32 64 128 256 256 128 96 96)
LAYERS = [("stage4 256->256", 256, 0, 256, 4), ("up1 256+128->256", 256, 128, 256, 3), ("up1 256->256", 256, 0, 256, 3),
          ("up2 128+64->128", 128, 64, 128, 2)]


def bench_coords(sigma, seed=5):
    z = np.load(os.path.join(ROOT, "tests", "golden", "step_synth180k.npz"))
    pts = torch.tensor(z["part"]).repeat(10, 1).float()
    g = torch.Generator().manual_seed(seed)
    pts = pts + sigma * torch.randn(pts.shape, generator=g)
    return torch.cat([torch.zeros(pts.shape[0], 1), torch.round(pts / 0.05)], 1)


def mma_rows(mask, perm, n_rows, rmask):
    m = mask[perm[:n_rows]] & rmask
    tot = 0
    for t in range(0, n_rows, 128):
        tot += 128 * bin(int(np.bitwise_or.reduce(m[t:t + 128]))).count("1")
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_offset_split: needs a CUDA device")
    h = _lib.get_handle(DEV)
    out = dict(device=torch.cuda.get_device_name(0), rows=[])
    for sigma in (1.0, 0.2, 0.05):
        coords = bench_coords(sigma)
        N = coords.shape[0]
        g = Geometry(h, N)
        g.split_groups = {2: {2, 3}, 3: {2, 3}, 4: {2, 3}}
        g.build(coords.to(DEV).contiguous(), N)
        torch.cuda.synchronize()
        rows = g.sizes()
        part = torch.zeros(2, N, 256, device=DEV)
        for name, c1, c2, cout, lvl in LAYERS:
            nbr = g.nbr3[lvl]
            M = rows[lvl]
            mask_t = g.mask_of[nbr.data_ptr()]
            mask = mask_t[:N].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
            gen = torch.Generator().manual_seed(c1 + cout)
            W = (torch.randn(27, c1 + c2, cout, generator=gen) / np.sqrt((c1 + c2) * 27)).to(DEV)
            Wp = h.pack_weights(W)
            A = torch.randn(2, N, 2 * c1, generator=gen).half().to(DEV)          # split companions, as the engine's lean activations
            B = torch.randn(2, N, 2 * c2, generator=gen).half().to(DEV) if c2 else None
            o = torch.zeros(2, N, 2 * cout, dtype=torch.float16, device=DEV)
            sc_, sh_ = torch.ones(cout, device=DEV), torch.zeros(cout, device=DEV)
            d = ConvDesc()
            d.c1, d.c2, d.cout, d.kvol = c1, c2, cout, 27
            d.weight, d.weight_packed = W.data_ptr(), Wp.data_ptr()
            d.scale, d.shift, d.relu = sc_.data_ptr(), sh_.data_ptr(), 1
            d.nbr, d.nbr_stride, d.mout_cap, d.npass = nbr.data_ptr(), N, N, 2
            d.row_mask = mask_t.data_ptr()
            for p in range(2):
                io = ConvIO()
                io.in1_h, io.in2_h, io.out_h = A[p].data_ptr(), (B[p].data_ptr() if B is not None else None), o[p].data_ptr()
                d.io[p] = io
            launches, issued = {}, {}
            launches[1] = [(0, 0, g.perm3[lvl], g.d_n[lvl], g.tile_order_of[nbr.data_ptr()][0])]
            issued[1] = mma_rows(mask, g.perm3[lvl].cpu().numpy(), M, (1 << 27) - 1)
            for G in (2, 3):
                launches[G], issued[G] = [], 0
                for k0, k1, perm_r, live_r, to_r in g.range_of[(nbr.data_ptr(), G)]:
                    launches[G].append((k0, k1, perm_r, g.d_n[lvl] if k1 == 27 else live_r, to_r))
                    n_r = M if k1 == 27 else int(live_r.item())
                    issued[G] += mma_rows(mask, perm_r.cpu().numpy(), n_r, ((1 << k1) - 1) & ~((1 << k0) - 1))

            def run(G):
                for k0, k1, perm_r, dm, to_r in launches[G]:
                    d.row_perm, d.tile_order128, d.d_mout = perm_r.data_ptr(), to_r.data_ptr(), dm.data_ptr()
                    d.k0, d.k1 = k0, k1
                    d.partial_in = part.data_ptr() if k0 > 0 else None
                    d.partial_out = part.data_ptr() if 0 < k1 < 27 else None
                    h.spconv(d, _lib.ALGO_TC)

            for G in (1, 2, 3):
                run(G)
            torch.cuda.synchronize()
            times = {1: [], 2: [], 3: []}
            for _ in range(args.reps):
                for G in (1, 2, 3):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        run(G)
                    e1.record()
                    e1.synchronize()
                    times[G].append(e0.elapsed_time(e1) / args.iters)
            pairs = int(sum(bin(int(x)).count("1") for x in mask[:M]))
            for G in (1, 2, 3):
                r = dict(sigma=sigma, layer=name, level=lvl, rows=M, G=G, ms=float(np.median(times[G])), ms_all=[round(t, 4) for t in times[G]],
                         mma_rows=issued[G], mma_efficiency=pairs / issued[G], launches=len(launches[G]))
                out["rows"].append(r)
                print(f"sigma {sigma:4.2f}  {name:18s} L{lvl} M={M:6d}  G={G}: {r['ms']:.4f} ms/conv  MMA rows {issued[G]:9d} "
                      f"(eff {r['mma_efficiency']:.2f}, {issued[1] / issued[G]:.2f}x fewer than G=1)  runs {r['ms_all']}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
