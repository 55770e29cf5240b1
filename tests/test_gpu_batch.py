"""Batched completion on the GPU: B scans sharing every launch against B = 1, scan by scan.

The convolutions' results for a row depend on which rows share its tile (DESIGN.md §3, batched sampling), so a batch agrees with
B = 1 under the project's 1e-3 rule rather than bit for bit: per element |a - b| <= 1e-3 (|b| + rms(b)).

  * the cluster farthest point sampling equals lb2_farthest_point_sample on every scan of a ragged batch;
  * a batch's level rows and kernel-map pairs are the sums of its scans', and no pair joins two batches;
  * the batched engine's NN indices equal lb2_nn_match with the reference's batch_scale = 2 max(C);
  * each step's x_t, multistep x0 and guided eps agree with B = 1 runs (eager and graph-replayed, small scans and one 180k-point step);
  * DiffCompletion.complete_scans agrees with per-scan complete_scan (refined and diffusion clouds), carries the multistep state slot-wise
    with fresh=False and starts fresh when the batch size changes;
  * batches that cannot fit or leave the key range are refused before allocation.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def close(a, b, tol=1e-3, frac=0.0):
    """at most `frac` of the elements outside |a - b| <= tol (|b| + rms(b))"""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    if a.shape != b.shape:
        return False
    r = (a - b).abs() / (b.abs() + b.pow(2).mean().sqrt() + 1e-30)
    return float((r > tol).double().mean()) <= frac


def clouds_close(a, b, frac=0.01):
    """two completed clouds: survivor counts within 1 %; in both directions at most `frac` of the points farther from the other
    cloud than the rule's scale 1e-3 rms(|b|); and element-wise under the rule where the counts match"""
    from scipy.spatial import cKDTree
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if abs(a.shape[0] - b.shape[0]) > 0.01 * b.shape[0]:
        return False
    tol = 1e-3 * np.sqrt((b ** 2).sum(1).mean())
    for p, q in ((a, b), (b, a)):
        if (cKDTree(q).query(p)[0] > tol).mean() > frac:
            return False
    return a.shape != b.shape or close(a, b, frac=frac)


# ---- farthest point sampling ------------------------------------------------------------------------------------------------------
def _fps_cases():
    from lidiff_b200.synth import range_filter, synthetic_scan
    from test_gpu_fullsize import load_case
    part = load_case("000123")[0]["part"]                                    # the FPS'd points of the reference's 000123.ply
    full = [range_filter(synthetic_scan(s)) for s in (0, 1)]                  # benchmark-sized raw scans
    g = np.random.default_rng(3)
    dup = np.repeat(g.normal(0, 10, (700, 3)), 3, axis=0)                    # every point three times: ties everywhere
    return part, full, dup


def test_batched_fps_equals_single_scan_fps():
    from lidiff_b200 import _lib
    from lidiff_b200.preprocess import farthest_point_sample, farthest_point_sample_batched
    part, full, dup = _fps_cases()
    cap = _lib.get_handle(DEV).fps_batched_capacity()
    assert cap >= max(f.shape[0] for f in full), f"on-chip capacity {cap} below a benchmark scan"
    t = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV)
    batches = [([part, full[0], full[1], dup[:1500]], 1500),                  # ragged
               ([dup, dup[:2000] * 2.0], 2000),                               # n_samples == n for the second scan
               ([full[1]], 18000),                                            # B = 1
               ([full[0], part], 18000)]
    for scans, ns in batches:
        got = farthest_point_sample_batched([t(s) for s in scans], ns, ordered=False).cpu()
        assert got.shape == (len(scans), ns)
        for b, s in enumerate(scans):
            ref = farthest_point_sample(t(s), ns, ordered=False).cpu()
            assert torch.equal(got[b], ref), f"scan {b} of {len(scans)} ({s.shape[0]} points, {ns} samples)"


# ---- engine -------------------------------------------------------------------------------------------------------------------------
def _engine(sds, N, B, **kw):
    from lidiff_b200.engine import DenoiseEngine
    return DenoiseEngine(sds["enc"], sds["diff"], device=DEV, n_points=N, denoising_steps=50, batch=B, **kw)


def _inputs(scan, B, T, seed):
    s = scan.reshape(-1, 3).double()
    scans = [s * torch.tensor([1.0 if b % 2 == 0 else -1.0, 1.0, 1.0], dtype=s.dtype) for b in range(B)]   # odd slots mirrored
    g = torch.Generator().manual_seed(seed)
    x_init = torch.stack(scans).to(DEV)
    start = torch.randn(x_init.shape, generator=g).to(DEV)
    noise = torch.randn((T,) + tuple(x_init.shape), generator=g).to(DEV)
    return x_init, x_init + start, noise


def _trajectory(eng, x_init, x_feats, noise, graphs):
    """x_t and x0 state after every step, and the guided eps of step 0 (eager, on the start state)"""
    N = eng.cap
    eng.use_graphs = graphs
    st = eng.start(x_init, x_feats, fresh=True)
    eps = torch.empty((N, 3), device=DEV)
    xb, cb, x0 = torch.empty_like(st["xa"]), torch.empty_like(st["ca"]), torch.zeros_like(st["x0s"])
    eng.step(0, st["xa"], xb, st["ca"], cb, st["x_init"], noise[0].reshape(N, 3).contiguous(), x0, eps_out=eps)
    geo = (eng.geom.sizes(), eng.geom.pairs[:13].cpu().clone(), [eng.geom.C[l][:n].clone() for l, n in enumerate(eng.geom.sizes())],
           [eng.geom.nbr3[l][:, :n].clone() for l, n in enumerate(eng.geom.sizes())])
    st = eng.start(x_init, x_feats, fresh=True)
    out = []
    for i in range(noise.shape[0]):
        eng.advance(st, noise[i].reshape(N, 3).contiguous())
        out.append((st["xa"].clone(), st["x0s"].clone()))
    torch.cuda.synchronize()
    return eps, out, geo


@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_batched_steps_equal_single_scan_steps(small_scan, calibrated_sds, B, graphs):
    N, T = small_scan.shape[1], 3
    x_init, x_feats, noise = _inputs(small_scan, B, T, 40 + B)
    eps_b, traj_b, (rows_b, pairs_b, C_b, nbr_b) = _trajectory(_engine(calibrated_sds, N, B), x_init, x_feats, noise, graphs)
    e1 = _engine(calibrated_sds, N, 1)
    rows_sum, pairs_sum = [0] * 5, torch.zeros(13, dtype=torch.int64)
    for b in range(B):
        eps_1, traj_1, (rows_1, pairs_1, _, _) = _trajectory(e1, x_init[b:b + 1], x_feats[b:b + 1], noise[:, b:b + 1], graphs)
        rows_sum = [r + q for r, q in zip(rows_sum, rows_1)]
        pairs_sum += pairs_1
        sl = slice(b * N, (b + 1) * N)
        assert close(eps_b[sl], eps_1), f"slot {b}: guided eps"
        # x0 = (x_t - x_init - sigma eps) / alpha magnifies eps by 1 / alpha (~14 at t = 999): once a point's voxel differs
        # between the runs, its x0 leaves the rule, so the x0 state is held to it at step 0 only
        assert close(traj_b[0][1][sl], traj_1[0][1], frac=0.01), f"slot {b}: x0 state"
        for i in range(T):
            assert close(traj_b[i][0][sl], traj_1[i][0], frac=0.01), f"slot {b}, step {i}: x_t"
    assert rows_b == rows_sum
    assert torch.equal(pairs_b, pairs_sum)
    for C, nbr in zip(C_b, nbr_b):                                           # no 3^3 pair joins two batches
        k = nbr >= 0
        src = C[:, 0][None].expand_as(nbr)[k]
        assert torch.equal(C[nbr[k].long(), 0], src)


def test_batched_nn_indices_equal_nn_match_with_the_reference_batch_scale(small_scan, calibrated_sds):
    N = small_scan.shape[1]
    x_init, x_feats, noise = _inputs(small_scan, 3, 1, 7)
    eng = _engine(calibrated_sds, N, 3)
    eng.use_graphs = False
    st = eng.start(x_init, x_feats, fresh=True)
    eng.advance(st, noise[0].reshape(-1, 3).contiguous())
    g = eng.geom
    for l, n in enumerate(g.sizes()):
        ref = torch.empty(n, dtype=torch.int32, device=DEV)
        scale = 2 * int(g.C[l][:n].max())                                    # minkunet.py match_part_to_full: 2 max(C)
        eng.h.nn_match(g.C[l][:n].contiguous(), None, n, eng.part_C, eng.part_dn, eng.part_cap, scale, ref)
        assert torch.equal(eng._bufs[f"nn{l}"][:n], ref), f"level {l}"


def test_one_full_size_batched_step_equals_single_scan_steps():
    from test_gpu_fullsize import load_case
    _, sds, scan, _, _, _ = load_case("synth180k")
    N = scan.shape[1]
    x_init, x_feats, noise = _inputs(scan, 2, 1, 5)
    eps_b, traj_b, _ = _trajectory(_engine(sds, N, 2), x_init, x_feats, noise, False)
    e1 = _engine(sds, N, 1)
    for b in range(2):
        eps_1, traj_1, _ = _trajectory(e1, x_init[b:b + 1], x_feats[b:b + 1], noise[:, b:b + 1], False)
        sl = slice(b * N, (b + 1) * N)
        assert close(eps_b[sl], eps_1) and close(traj_b[0][0][sl], traj_1[0][0]) and close(traj_b[0][1][sl], traj_1[0][1])


# ---- whole scans ----------------------------------------------------------------------------------------------------------------------
def _pipe(sds, N, T=3):
    from lidiff_b200.pipeline import DiffCompletion
    return DiffCompletion(state_dicts=sds, denoising_steps=T, device=DEV, hparams={"data": {"num_points": N}})


def test_complete_scans_equals_per_scan_complete_scan(small_scan, calibrated_sds):
    N = small_scan.shape[1]
    x_init, _, noise = _inputs(small_scan, 2, 3, 9)
    x2, _, noise2 = _inputs(small_scan, 3, 3, 10)
    start = torch.randn(x_init.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    start2 = torch.randn(x2.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    pipe = _pipe(calibrated_sds, N)
    first = pipe.complete_scans(list(x_init), start_noise=start, step_noise=noise, preprocessed=True, fresh=True)
    carried = pipe.complete_scans(list(x_init.flip(0)), start_noise=start, step_noise=noise, preprocessed=True)   # fresh=False
    restarted = pipe.complete_scans(list(x_init.flip(0)), start_noise=start, step_noise=noise, preprocessed=True, fresh=True)
    resized = pipe.complete_scans(list(x2), start_noise=start2, step_noise=noise2, preprocessed=True)              # B 2 -> 3: fresh
    for b in range(2):
        one = _pipe(calibrated_sds, N)
        r1 = one.complete_scan(x_init[b:b + 1], start_noise=start[b], step_noise=noise[:, b], preprocessed=True, fresh=True)
        r2 = one.complete_scan(x_init.flip(0)[b:b + 1], start_noise=start[b], step_noise=noise[:, b], preprocessed=True, fresh=False)
        for k, what in ((0, "refined"), (1, "diffusion")):
            assert clouds_close(first[b][k], r1[k]), f"scan {b}: {what} cloud"
            # the carried x0 already drifted in the points whose voxel differs (see above): counts here; the slot-wise carry itself
            # is checked bit for bit on the CPU stand-ins (tests/test_batch_host.py)
            assert abs(carried[b][k].shape[0] - r2[k].shape[0]) <= 0.01 * r2[k].shape[0], f"scan {b}: {what} cloud, carried state"
            assert not np.array_equal(carried[b][k], restarted[b][k]), f"scan {b}: the carried state changed nothing"
    for b in range(3):
        r = _pipe(calibrated_sds, N).complete_scan(x2[b:b + 1], start_noise=start2[b], step_noise=noise2[:, b], preprocessed=True,
                                                   fresh=True)
        assert clouds_close(resized[b][0], r[0]) and clouds_close(resized[b][1], r[1]), f"scan {b} after the batch size changed"


def test_a_short_batch_releases_the_engine_of_the_long_one(small_scan, calibrated_sds):
    import weakref
    N = small_scan.shape[1]
    x3, _, n3 = _inputs(small_scan, 3, 3, 11)
    pipe = _pipe(calibrated_sds, N)
    pipe.complete_scans(list(x3), step_noise=n3, preprocessed=True)
    eng3 = weakref.ref(pipe._engine)
    torch.cuda.synchronize()
    with_3 = torch.cuda.memory_allocated(DEV)
    pipe.complete_scans(list(x3[:2]), step_noise=n3[:, :2], preprocessed=True)
    torch.cuda.synchronize()
    assert eng3() is None and pipe._engine.B == 2
    assert torch.cuda.memory_allocated(DEV) < with_3


def test_engine_refuses_batches_that_cannot_fit(calibrated_sds):
    with pytest.raises(RuntimeError, match="device memory"):
        _engine(calibrated_sds, 180000, 200)
    with pytest.raises(RuntimeError, match="device memory"):          # ~117 KB per row: 4 x 180 000 rows exceed an 80 GB card
        _engine(calibrated_sds, 180000, 4)
    with pytest.raises(RuntimeError, match="10 batch bits"):
        _engine(calibrated_sds, 16, 1025)
