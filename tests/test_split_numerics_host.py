"""The bars of tests/test_gpu_conv_numerics.py have teeth, checked without a GPU: an emulation of FP16x3 as the kernel forms it
(restated split, 2^k weight pre-scale, fp32 sums) passes them on every case, and two cheaper splits fail the statistical bar
(tests/split_numerics.py holds the error model).  Also pins the host restatement of the split against an independent one and the
CPU fake backend's companions against it."""
import numpy as np
import pytest
import torch

import split_numerics as sn

MUTANT_CASES = [c for c in sn.CASES if c[4] >= -4]          # below, the 2^-25 floor hides a dropped cross term by design


@pytest.fixture(scope="module")
def refs():
    return {}


def _ref(refs, c):
    if c not in refs:
        X, W = sn.case_operands(c)
        refs[c] = (X, W, sn.Reference(c, X, W))
    return refs[c]


@pytest.mark.parametrize("c", sn.CASES, ids=sn.case_id)
def test_fp16x3_emulation_passes_both_bars(refs, c):
    X, W, ref = _ref(refs, c)
    eh, es = ref.errors(sn.emulate(c, X, W, "f16x3"))
    print(f"{sn.case_id(c)}: hard {eh:.3f} of bound, stat {es:.2e} (tau_s {sn.tau_s(ref.ctot, ref.kvol):.2e})")
    assert eh <= 1.0
    assert es <= sn.tau_s(ref.ctot, ref.kvol)


@pytest.mark.parametrize("scheme", ["f16x2", "f16x3_last"])
@pytest.mark.parametrize("c", MUTANT_CASES, ids=sn.case_id)
def test_cheaper_splits_fail_the_statistical_bar(refs, c, scheme):
    if scheme == "f16x3_last" and (c[0] + c[1]) % 64 == 0:
        pytest.skip("no partial last chunk: the mutant is FP16x3")
    X, W, ref = _ref(refs, c)
    _, es = ref.errors(sn.emulate(c, X, W, scheme))
    t = sn.tau_s(ref.ctot, ref.kvol)
    print(f"{sn.case_id(c)} {scheme}: stat {es:.2e} = {es / t:.1f} x tau_s")
    assert es > t


def _split_np(x):
    """independent restatement: numpy's fp16 cast, the saturation of hi by hand"""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        hi = x.astype(np.float16)
        hi = np.where(np.isinf(hi), np.sign(x) * np.float16(65504), hi).astype(np.float16)
        r = (x - hi.astype(np.float32)).astype(np.float32)
        lo = r.astype(np.float16)
    return hi, lo


def _bits_cases():
    g = torch.Generator().manual_seed(9)
    rnd = torch.randint(-2 ** 31, 2 ** 31, (1 << 20,), generator=g, dtype=torch.int64).to(torch.int32).view(torch.float32)
    return torch.cat([sn.edge_values(), rnd])


def test_restated_split_equals_independent_restatement():
    x = _bits_cases()
    hi, lo = sn.split(x)
    nh, nl = _split_np(x.numpy())
    assert sn.same_bits(hi, torch.from_numpy(nh)) and sn.same_bits(lo, torch.from_numpy(nl))
    e = sn.edge_values()
    h, l = sn.split(e)
    for v, a, b in zip(e.tolist(), h.tolist(), l.tolist()):          # the contract's named cases
        if np.isnan(v):
            assert np.isnan(a) and np.isnan(b)
        elif abs(v) >= 65504:                                          # hi saturates; lo is +-inf from 131024 on, +-inf included
            assert abs(a) == 65504.0 and np.isinf(b) == (abs(v) >= 131024.0)
        else:
            assert abs(a + b - v) <= 2.0 ** -22 * abs(v) + 2.0 ** -25


def test_fake_backend_companions_follow_the_split():
    import fake_backend
    h = fake_backend.FakeHandle()
    x = _bits_cases()[:4096].reshape(-1, 16).contiguous()
    out, out_h = torch.empty_like(x), torch.zeros(x.shape[0], 32, dtype=torch.float16)
    h.gate_mul(x, torch.ones(1, 16), None, None, x.shape[0], 16, out, out_h)
    hi, lo = sn.split(x)
    assert sn.same_bits(out_h[:, :16], hi) and sn.same_bits(out_h[:, 16:], lo)
    buf = torch.zeros(x.shape[0], 32, dtype=torch.float16)
    fake_backend._write_act(None, buf.data_ptr(), x.shape[0], 16, x.double())
    assert sn.same_bits(buf[:, :16], hi) and sn.same_bits(buf[:, 16:], lo)
