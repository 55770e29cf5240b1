"""The restatements and the error model of tests/dense_numerics.py on the CPU: the FPS and nearest-neighbour restatements agree
with oracle/ on ties, duplicates and single points; a numpy fp32 emulation of each dense kernel's summation order stays within
the model's bound over the shape grid of tests/test_gpu_dense_edges.py, and emulations with TF32 operands, a dropped k-tile or a
dropped hidden unit leave it (so the bound is neither wrong nor loose enough to hide those)."""
import numpy as np
import pytest
import torch

import dense_numerics as dn
from oracle import me_cpu as ome
from oracle.pipeline import farthest_point_sample as fps_oracle

LIN_N_IN = [1, 15, 16, 17, 256, 512]
LIN_N_OUT = [1, 3, 63, 64, 65, 256]
HEAD_N_IN = list(range(16, 129, 16))
HEAD_N_HID = [1, 20, 64]
HEAD_N_OUT = [1, 3, 4, 5, 18, 24]


# ---- farthest point sampling -------------------------------------------------------------------------------------------------
def _fps_clouds():
    g = np.random.default_rng(0)
    lat = np.stack(np.meshgrid(np.arange(6), np.arange(5), np.arange(4), indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    dup = np.repeat(g.normal(size=(40, 3)), 5, axis=0)
    return {
        "single": (np.array([[1.0, 2.0, 3.0]]), 1),
        "pair": (np.array([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]]), 2),
        "identical": (np.full((50, 3), 7.25), 50),
        "lattice": (lat[g.permutation(lat.shape[0])], lat.shape[0]),
        "duplicates": (dup[g.permutation(dup.shape[0])], 120),
        "offset": (g.normal(size=(500, 3)) + 1e6, 200),
        "gauss": (g.normal(size=(2000, 3)) * 10, 300),
    }


@pytest.mark.parametrize("case", list(_fps_clouds()))
def test_fps_sequence_restates_the_oracle(case):
    p, ns = _fps_clouds()[case]
    seq = dn.fps_sequence(p, ns)
    assert np.array_equal(np.sort(seq), fps_oracle(p, ns))
    assert seq[0] == 0 and len(set(seq.tolist())) == min(ns, np.unique(p, axis=0).shape[0])
    if case == "identical":                         # every running minimum is 0: the first index wins every step
        assert (seq == 0).all()


@pytest.mark.parametrize("case", ["lattice", "duplicates", "gauss"])
def test_fps_torch_form_equals_the_numpy_form(case):
    p, ns = _fps_clouds()[case]
    other = _fps_clouds()["offset"][0]
    got = dn.fps_sequence_torch([torch.tensor(p), torch.tensor(other)], min(ns, other.shape[0]))
    assert np.array_equal(got[0].numpy(), dn.fps_sequence(p, min(ns, other.shape[0])))
    assert np.array_equal(got[1].numpy(), dn.fps_sequence(other, min(ns, other.shape[0])))


# ---- nearest neighbour ---------------------------------------------------------------------------------------------------------
def _nn_sets():
    g = np.random.default_rng(1)
    k = np.concatenate([np.zeros((300, 1), np.int64), g.integers(-8, 8, (300, 3)) * 16], 1)       # many duplicates
    q = np.concatenate([np.zeros((2000, 1), np.int64), g.integers(-200, 200, (2000, 3))], 1)
    k2, q2 = k.copy(), q.copy()
    k2[150:, 0], q2[1000:, 0] = 1, 1
    one = np.array([[0, 5, -3, 2]])
    return {"ties": (q, k), "batches": (q2, k2), "single": (q, one), "single_query": (one, k)}


@pytest.mark.parametrize("case", list(_nn_sets()))
def test_nn_brute_restates_the_oracle(case):
    q, k = _nn_sets()[case]
    ref = ome.match_part_to_full(torch.tensor(q), torch.tensor(k)).numpy()
    assert np.array_equal(dn.nn_brute(q, k), ref)


def test_nn_brute_ties_take_the_lowest_index():
    k = np.array([[0, 2, 0, 0], [0, -2, 0, 0], [0, 2, 0, 0], [1, 0, 0, 0]])
    q = np.array([[0, 0, 0, 0], [0, 2, 0, 0], [1, 5, 0, 0], [2, 0, 0, 0]])
    assert dn.nn_brute(q, k).tolist() == [0, 0, 3, 3]


# ---- dense layers ----------------------------------------------------------------------------------------------------------------
def _linear_operands(m, n_in, n_out, seed, structured=False):
    g = np.random.default_rng(seed)
    if structured:      # every operand rounds down under TF32 by 3 * 2^-13 relative: the errors add up instead of cancelling
        v = np.float32(1 + 3 * 2.0 ** -13)
        return np.full((m, n_in), v, np.float32), np.full((n_out, n_in), v, np.float32), np.zeros(n_out, np.float32)
    return (g.standard_normal((m, n_in)).astype(np.float32), (g.standard_normal((n_out, n_in)) * 0.1).astype(np.float32),
            g.standard_normal(n_out).astype(np.float32))


@pytest.mark.parametrize("n_in", LIN_N_IN)
@pytest.mark.parametrize("n_out", LIN_N_OUT)
def test_linear_emulation_within_the_bound_and_mutants_leave_it(n_in, n_out):
    m = 65
    x, w, b = _linear_operands(m, n_in, n_out, n_in * 1000 + n_out)
    g = np.random.default_rng(n_in + n_out)
    add = g.standard_normal((m, n_out)).astype(np.float32)
    pre = g.standard_normal(n_in).astype(np.float32)
    for act in (0, 1, 2):
        for kw in ({}, {"addend": add}, {"prebias": pre, "pre_act": 1}):
            ref, bound = dn.linear_reference(x, w, b, act=act, **kw)
            assert dn.within(dn.emulate_linear(x, w, b, act=act, **kw), ref, bound) <= 1.0, (act, list(kw))
    ref, bound = dn.linear_reference(x, w, b)
    assert dn.within(dn.emulate_linear(x, w, b, mutant="drop_tile"), ref, bound) > 1.0
    xs, ws, bs = _linear_operands(m, n_in, n_out, 0, structured=True)
    ref, bound = dn.linear_reference(xs, ws, bs)
    assert dn.within(dn.emulate_linear(xs, ws, bs), ref, bound) <= 1.0
    assert dn.within(dn.emulate_linear(xs, ws, bs, mutant="tf32"), ref, bound) > 1.0


def _head_operands(m, n_in, n_hid, n_out, seed, structured=False):
    g = np.random.default_rng(seed)
    if structured:
        v = np.float32(1 + 3 * 2.0 ** -13)
        return (np.full((m, n_in), v, np.float32), np.full((n_hid, n_in), v, np.float32), np.zeros(n_hid, np.float32),
                np.full((n_out, n_hid), v, np.float32), np.zeros(n_out, np.float32))
    return (g.standard_normal((m, n_in)).astype(np.float32), (g.standard_normal((n_hid, n_in)) / 10).astype(np.float32),
            g.standard_normal(n_hid).astype(np.float32), (g.standard_normal((n_out, n_hid)) / 4).astype(np.float32),
            g.standard_normal(n_out).astype(np.float32))


@pytest.mark.parametrize("n_in", HEAD_N_IN)
@pytest.mark.parametrize("n_hid", HEAD_N_HID)
def test_head_mlp_emulation_within_the_bound_and_mutants_leave_it(n_in, n_hid):
    m = 64
    for n_out in HEAD_N_OUT:
        ops = _head_operands(m, n_in, n_hid, n_out, n_in * 100 + n_hid + n_out)
        for act in (0, 2):
            ref, bound = dn.head_mlp_reference(*ops, out_act=act)
            assert dn.within(dn.emulate_head_mlp(*ops, out_act=act), ref, bound) <= 1.0, (n_out, act)
        ref, bound = dn.head_mlp_reference(*ops)
        assert dn.within(dn.emulate_head_mlp(*ops, mutant="drop_hidden"), ref, bound) > 1.0, n_out
        sops = _head_operands(m, n_in, n_hid, n_out, 0, structured=True)
        ref, bound = dn.head_mlp_reference(*sops)
        assert dn.within(dn.emulate_head_mlp(*sops), ref, bound) <= 1.0, n_out
        assert dn.within(dn.emulate_head_mlp(*sops, mutant="tf32"), ref, bound) > 1.0, n_out


def test_tf32_rounding_keeps_ten_mantissa_bits():
    v = np.array([1 + 3 * 2.0 ** -13, 1 + 2.0 ** -10, 1 + 2.0 ** -11, -(1 + 5 * 2.0 ** -12)], np.float32)
    assert dn.tf32(v).tolist() == [1.0, 1 + 2.0 ** -10, 1 + 2.0 ** -10, -(1 + 2.0 ** -10)]
