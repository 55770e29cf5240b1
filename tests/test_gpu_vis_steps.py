"""The denoising trajectory behind tools/vis_steps.py on the GPU: with random weights and injected noise (T = 5), the last panels
(post-processed and refined clouds) equal DiffCompletion.complete_scan(..., fresh=True) bit for bit, and the k-step snapshots
(DenoiseEngine.run(snapshot_steps=...), taken between graph replays) equal x_t of an eager start / advance loop."""
import numpy as np
import pytest
import torch

from lidiff_b200.synth import synthetic_scan

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, N = 5, 20_000


@pytest.fixture(scope="module")
def pipe():
    from lidiff_b200.pipeline import DiffCompletion
    from lidiff_b200.weights import random_state_dict
    sds = {k: random_state_dict(k, i) for i, k in enumerate(("enc", "diff", "refine"))}
    return DiffCompletion(state_dicts=sds, denoising_steps=T, device=DEV, hparams={"data": {"num_points": N}})


def test_trajectory_panels_equal_complete_scan_and_an_eager_loop(pipe):
    from lidiff_b200.render import Camera
    from lidiff_b200.tools import vis_steps
    raw = synthetic_scan(4)
    g = torch.Generator().manual_seed(11)
    start = torch.randn((1, N, 3), generator=g)
    noise = torch.randn((T, 1, N, 3), generator=g)
    steps = [0, 2, 5]
    traj = vis_steps.trajectory(pipe, raw, steps, start.to(DEV), noise.to(DEV))
    assert sorted(traj["steps"]) == steps and all(v.shape == (N, 3) for v in traj["steps"].values())

    refined, post = pipe.complete_scan(raw, start.to(DEV), noise.to(DEV), fresh=True)
    assert np.array_equal(traj["refined"].cpu().numpy(), refined) and np.array_equal(traj["post"].cpu().numpy(), post)

    eng = pipe.engine()
    pre = pipe.preprocess_scan(raw).to(DEV)
    assert torch.equal(traj["scan"], pre.reshape(-1, 3))
    use_graphs, eng.use_graphs = eng.use_graphs, False
    try:
        st = eng.start(pre, pre + start.to(DEV), fresh=True)
        assert torch.equal(st["xa"], traj["steps"][0])
        for i in range(T):
            eng.advance(st, noise[i].reshape(-1, 3).to(DEV).contiguous())
            if i + 1 in traj["steps"]:
                assert torch.equal(st["xa"], traj["steps"][i + 1]), f"snapshot after {i + 1} steps"
    finally:
        eng.use_graphs = use_graphs
    assert torch.equal(traj["steps"][T].cpu(), st["xa"].cpu())

    cam = Camera.fit(traj["scan"], width=64, height=48)
    img = vis_steps.strip(vis_steps.panels_of(traj), cam, (float(pre[..., 2].min()), float(pre[..., 2].max())))
    assert img.shape == (48, 64 * (len(steps) + 3), 3) and img.device.type == "cuda"


def test_snapshot_steps_outside_the_trajectory_are_refused(pipe):
    eng = pipe.engine()
    pre = pipe.preprocess_scan(synthetic_scan(4)).to(DEV)
    with pytest.raises(ValueError):
        eng.run(pre, pre, snapshot_steps=[T + 1])
