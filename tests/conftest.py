import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def make_scan(n_part=1500, seed=0, repeat=10):
    """Small KITTI-shaped conditioning scan (1, n_part*repeat, 3) float64, like preprocess_scan's output
    (random subsample instead of FPS to keep CPU tests fast)."""
    from lidiff_b200.synth import range_filter, synthetic_scan
    raw = range_filter(synthetic_scan(seed, beams=32, azimuths=512))
    g = np.random.default_rng(seed + 100)
    sel = np.sort(g.choice(raw.shape[0], n_part, replace=False))
    return torch.tensor(raw[sel]).repeat(repeat, 1)[None]


@pytest.fixture(scope="session")
def small_scan():
    return make_scan(1500, 0)


@pytest.fixture(scope="session")
def calibrated_sds(small_scan):
    from oracle.pipeline import calibrated_state_dicts
    return calibrated_state_dicts(small_scan, seed=0)
