"""CPU study (not collected by pytest; run `python scripts/numerics_split_study.py`) of how the operand split of the tensor-core
convolution propagates through the 49-layer guided U-Net of the oracle.  Every scheme replaces the per-offset GEMM of
oracle.me_cpu.conv by an emulation of the products the hardware would form (fp32 accumulation, RN — the tensor-core truncation of the
real kernels is a separate, measured effect, DESIGN.md §3), and reports the error of the guided eps against the fp64 network with
the metric of tests/test_gpu_networks.py: max |a - b| / (|b| + rms(b)).
Schemes:  fp32           plain fp32 GEMM (what the FFMA kernel and ME compute)
          f16x3          A_hi.W_hi + A_lo.W_hi + A_hi.W_lo, fp16 operands           (shipped)
          f16x2a / x2w   one cross term dropped (A_lo.W_hi kept / A_hi.W_lo kept)
          f16x1          A_hi.W_hi only
          f16+f8x2       A_hi.W_hi in fp16, both cross terms with e4m3 operands (kind::f8f6f4 at twice the fp16 rate): 2 MMA units
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle.me_cpu as ome  # noqa: E402
from oracle.pipeline import DiffCompletionOracle, calibrated_state_dicts  # noqa: E402
from conftest import make_scan  # noqa: E402

F8 = torch.float8_e4m3fn


def q16(x):
    return x.clamp(-65504.0, 65504.0).half().float()


def q8(x):
    return x.clamp(-448.0, 448.0).to(F8).float()


def pow2_scale(w, target):
    m = float(w.abs().max())
    return 2.0 ** np.floor(np.log2(target / m)) if m > 0 else 1.0


def gemm(a, w, scheme):
    if scheme == "fp64":
        return a.double() @ w.double()
    a, w = a.float(), w.float()
    if scheme == "fp32":
        return a @ w
    s = pow2_scale(w, 32768.0)                      # weights pre-scaled into the fp16 range (lb2_pack_weights)
    ws = w * s
    a_hi, w_hi = q16(a), q16(ws)
    a_lo, w_lo = a - a_hi, ws - w_hi
    out = a_hi @ w_hi
    if scheme == "f16x3":
        out = out + q16(a_lo) @ w_hi + a_hi @ q16(w_lo)
    elif scheme == "f16x2a":
        out = out + q16(a_lo) @ w_hi
    elif scheme == "f16x2w":
        out = out + a_hi @ q16(w_lo)
    elif scheme == "f16+f8x2":
        sa = pow2_scale(a, 256.0) if a.numel() else 1.0            # per-tensor activation scale for the e4m3 copy of A
        out = out + (q8(a_lo * 2048.0 * sa) @ q8(ws / 2048.0)) / sa      # A_lo.W : A_lo*2^11 and W*2^-11 both sit in e4m3's range
        out = out + (q8(a * sa) @ q8(w_lo)) / sa                          # A.W_lo : |W_lo| <= 2^-11 * 32768 = 16 already fits
    elif scheme != "f16x1":
        raise ValueError(scheme)
    return out / s


def patched_conv(scheme):
    def conv(x, W, ks, stride=1, transposed=False):
        dt = torch.float64 if scheme == "fp64" else torch.float32
        if W.dim() == 2:
            return x.replace(gemm(x.F, W, scheme).to(dt))
        ts_out = x.ts // stride if transposed else x.ts * stride
        maps = x.geom.kernel_map(x.ts, ks, stride, transposed)
        m_out = x.geom.stride_level(ts_out).shape[0]
        out = torch.zeros(m_out, W.shape[2], dtype=dt)
        for k, (i_rows, o_rows) in enumerate(maps):
            if i_rows.shape[0]:
                out.index_add_(0, torch.from_numpy(o_rows), gemm(x.F[torch.from_numpy(i_rows)], W[k], scheme).to(dt))
        return ome.SparseTensor(out, x.geom, ts_out)
    return conv


def guided_eps(sds, scan, start, scheme):
    orig = ome.conv
    ome.conv = patched_conv(scheme)
    try:
        fp64 = scheme == "fp64"
        o = DiffCompletionOracle(sds["enc"], sds["diff"], sds["refine"], denoising_steps=50, dtype=torch.float64 if fp64 else torch.float32)
        x_t, x_c, x_u = o.points_to_tensor(scan + start), o.points_to_tensor(scan), o.points_to_tensor(torch.zeros_like(scan))
        o.dpm.set_timesteps(o.dpm.num_inference_steps)
        return o.classfree_forward(x_t, x_c, x_u, o.dpm.timesteps[0][None]).double()
    finally:
        ome.conv = orig


def rel_err(a, b):
    return float(((a - b).abs() / (b.abs() + b.pow(2).mean().sqrt())).max())


def main():
    scan = make_scan(int(os.environ.get("STUDY_POINTS", 600)), 0)
    sds = calibrated_state_dicts(scan, seed=0)
    start = torch.randn(scan.shape, generator=torch.Generator().manual_seed(5), dtype=scan.dtype)
    ref = guided_eps(sds, scan, start, "fp64")
    print(f"{scan.shape[1]} points; guided eps rms {float(ref.pow(2).mean().sqrt()):.3e}")
    for scheme in ("fp32", "f16x3", "f16+f8x2", "f16x2a", "f16x2w", "f16x1"):
        print(f"  {scheme:10s} rel err vs fp64 network: {rel_err(guided_eps(sds, scan, start, scheme), ref):.3e}")


if __name__ == "__main__":
    main()
