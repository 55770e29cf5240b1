"""Batched completion without a GPU: DiffCompletion.complete_scans (operator path and fused engine) against per-scan
complete_scan on the CPU stand-ins of tests/fake_backend.py, the grouping of a rank's scans into batches, the engine's refusals,
and the completion CLI's --batch-size output."""
import numpy as np
import pytest
import torch
from click.testing import CliRunner

import fake_backend
from conftest import make_scan
from oracle.pipeline import calibrated_state_dicts


@pytest.fixture(scope="module")
def pair():
    s = make_scan(250, 3)
    scans = [s, s * torch.tensor([-1.0, 1.0, 1.0], dtype=s.dtype)]     # two different (1, 2500, 3) scans (the second mirrored)
    sds = calibrated_state_dicts(scans[0], seed=5)
    g = torch.Generator().manual_seed(21)
    N = scans[0].shape[1]
    return dict(scans=scans, sds=sds, N=N, start=torch.randn((2, N, 3), generator=g), noise=torch.randn((2, 2, N, 3), generator=g))


def _pipe(pair, engine):
    from lidiff_b200.pipeline import DiffCompletion
    return DiffCompletion(state_dicts=pair["sds"], denoising_steps=2, device="cpu", hparams={"data": {"num_points": pair["N"]}},
                          engine=engine)


@pytest.mark.parametrize("engine", [False, True], ids=["operators", "engine"])
def test_complete_scans_equals_per_scan_complete_scan(pair, monkeypatch, engine):
    fake_backend.install(monkeypatch)
    pipe = _pipe(pair, engine)
    got = pipe.complete_scans([s[0] for s in pair["scans"]], start_noise=pair["start"], step_noise=pair["noise"], preprocessed=True,
                              fresh=True)
    assert len(got) == 2
    for b in range(2):
        ref = pipe.complete_scan(pair["scans"][b], start_noise=pair["start"][b], step_noise=pair["noise"][:, b], preprocessed=True,
                                 fresh=True)
        if engine:      # the engine's stand-in kernels are row-local: bit-identical
            assert np.array_equal(got[b][1], ref[1]), f"scan {b}: diffusion cloud"
            assert np.array_equal(got[b][0], ref[0]), f"scan {b}: refined cloud"
        else:           # the operator surface runs some layers as torch CPU matmuls whose blocking depends on the row count
            for k, what in ((1, "diffusion"), (0, "refined")):
                assert got[b][k].shape == ref[k].shape, f"scan {b}: {what} cloud"
                assert np.abs(got[b][k] - ref[k]).max() < 1e-4, f"scan {b}: {what} cloud"


def test_batch_size_change_starts_fresh(pair, monkeypatch):
    """fresh=False carries the multistep state between batches of one size only: after a batch of 2, a batch of 1 equals a fresh run"""
    fake_backend.install(monkeypatch)
    pipe = _pipe(pair, True)
    scans = [s[0] for s in pair["scans"]]
    pipe.complete_scans(scans, start_noise=pair["start"], step_noise=pair["noise"], preprocessed=True, fresh=True)
    carried = pipe.complete_scans(scans[:1], start_noise=pair["start"][:1], step_noise=pair["noise"][:, :1], preprocessed=True)
    fresh = pipe.complete_scan(pair["scans"][0], start_noise=pair["start"][0], step_noise=pair["noise"][:, 0], preprocessed=True,
                               fresh=True)
    assert np.array_equal(carried[0][1], fresh[1])


def test_fresh_false_carries_each_slots_multistep_state(pair, monkeypatch):
    """two batches of the same size with fresh=False: slot b of the second equals complete_scan(fresh=False) of scan b after
    complete_scan(fresh=True) of the first batch's scan b (the engine's stand-in kernels are row-local: bit-identical)"""
    fake_backend.install(monkeypatch)
    first, second = [s[0] for s in pair["scans"]], [s[0] for s in pair["scans"][::-1]]
    pipe = _pipe(pair, True)
    pipe.complete_scans(first, start_noise=pair["start"], step_noise=pair["noise"], preprocessed=True, fresh=True)
    got = pipe.complete_scans(second, start_noise=pair["start"], step_noise=pair["noise"], preprocessed=True, fresh=False)
    fresh = pipe.complete_scans(second, start_noise=pair["start"], step_noise=pair["noise"], preprocessed=True, fresh=True)
    for b in range(2):
        one = _pipe(pair, True)
        one.complete_scan(first[b][None], start_noise=pair["start"][b], step_noise=pair["noise"][:, b], preprocessed=True, fresh=True)
        ref = one.complete_scan(second[b][None], start_noise=pair["start"][b], step_noise=pair["noise"][:, b], preprocessed=True,
                                fresh=False)
        assert np.array_equal(got[b][1], ref[1]) and np.array_equal(got[b][0], ref[0]), f"slot {b}"
        assert not np.array_equal(got[b][1], fresh[b][1]), f"slot {b}: the carried state changed nothing"


def test_one_engine_alive_across_batch_sizes(pair, monkeypatch):
    """B, B, then a short batch: the short batch releases the engine of B instead of building a second one next to it"""
    import weakref
    fake_backend.install(monkeypatch)
    pipe = _pipe(pair, True)
    scans = [s[0] for s in pair["scans"]]
    kw = dict(start_noise=pair["start"], step_noise=pair["noise"], preprocessed=True)
    pipe.complete_scans(scans, **kw)
    eng2 = pipe._engine
    pipe.complete_scans(scans, **kw)
    assert pipe._engine is eng2 and eng2.B == 2
    ref = weakref.ref(eng2)
    del eng2
    pipe.complete_scans(scans[:1], start_noise=pair["start"][:1], step_noise=pair["noise"][:, :1], preprocessed=True)
    assert ref() is None and pipe._engine.B == 1


def test_batches_of_rank_group_every_scan_once_in_order():
    from lidiff_b200.sharding import batches_of_rank, scans_of_rank
    for n, world, batch in [(0, 1, 2), (7, 1, 2), (7, 2, 3), (10, 3, 4), (5, 8, 1), (9, 2, 1)]:
        for rank in range(world):
            groups = batches_of_rank(n, world, rank, batch)
            assert [b for g in groups for b in g] == scans_of_rank(n, world, rank)
            assert all(len(g) == batch for g in groups[:-1]) and all(1 <= len(g) <= batch for g in groups)
    with pytest.raises(ValueError):
        batches_of_rank(4, 1, 0, 0)


def test_engine_refuses_batches_outside_the_key_range():
    from lidiff_b200.engine import DenoiseEngine
    for b in (0, -1, 1025):
        with pytest.raises(RuntimeError, match="batch"):
            DenoiseEngine({}, {}, device="cpu", n_points=16, batch=b)
    with pytest.raises(RuntimeError, match="32-bit"):
        DenoiseEngine({}, {}, device="cpu", n_points=180000, batch=1000)


class _StubCompletion:
    """stands in for lidiff_b200.pipeline.DiffCompletion: a (refined, diffusion) pair that depends on the scan alone, as the real
    one's does when the noise of each scan is fixed"""

    def __init__(self, *a, **k):
        self.batches = []

    def complete_scan(self, points):
        self.batches.append(1)
        g = np.random.default_rng(points.shape[0])
        post = points[: points.shape[0] // 2] + g.normal(0, 0.01, (points.shape[0] // 2, 3))
        return (post[:, None, :] + g.normal(0, 0.03, (post.shape[0], 6, 3))).reshape(-1, 3), post

    def complete_scans(self, scans):
        out = [self.complete_scan(p) for p in scans]
        self.batches[-len(scans):] = [len(scans)]
        return out


def _run_cli(monkeypatch, tmp_path, scans, extra):
    from lidiff_b200.tools import diff_completion_pipeline as P
    stub = _StubCompletion()
    monkeypatch.setattr(P, "DiffCompletion", lambda *a, **k: stub)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    out = tmp_path / "out"
    res = CliRunner().invoke(P.main, ["--path", str(scans), "--out", str(out), "-T", "2"] + extra, catch_exceptions=False)
    assert res.exit_code == 0, res.output
    return out / "diff_net_T2_s6.0", stub.batches


def test_cli_batch_size_writes_the_same_files(monkeypatch, tmp_path):
    from lidiff_b200.synth import synthetic_scan
    scans = tmp_path / "scans"
    scans.mkdir()
    for b in range(5):
        np.c_[synthetic_scan(b, beams=8, azimuths=64 + 8 * b), np.ones(512 + 64 * b)].astype(np.float32).tofile(scans / f"{b:06d}.bin")
    one, n1 = _run_cli(monkeypatch, tmp_path / "a", scans, [])
    two, n2 = _run_cli(monkeypatch, tmp_path / "b", scans, ["--batch-size", "2"])
    assert n1 == [1] * 5 and n2 == [2, 2, 1]
    for kind in ("refine", "diff"):
        names = sorted(p.name for p in (one / kind).iterdir())
        assert names == sorted(p.name for p in (two / kind).iterdir()) == [f"{b:06d}.ply" for b in range(5)]
        for nm in names:
            assert (one / kind / nm).read_bytes() == (two / kind / nm).read_bytes()
