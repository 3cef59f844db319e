import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for it in items:
        if 'gpu' in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope='session')
def seeded_sd():
    from patch2pix_b200.synth import make_seeded_state_dict
    return make_seeded_state_dict(0)


@pytest.fixture(scope='session')
def consensus_sd():
    """Benchmark-workload weights: as seeded_sd but with trained-like (centre-dominant) NC filters."""
    from patch2pix_b200.synth import make_seeded_state_dict
    return make_seeded_state_dict(0, nc_init='consensus')
