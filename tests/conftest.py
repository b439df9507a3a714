import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


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
def port():
    from oracle.oracle import Port
    return Port()


@pytest.fixture(scope='session')
def scene():
    """Seeded lego-like occupancy scene + 4096 spiral-view rays."""
    from xrnerf_b200 import synth
    grid = synth.lego_like_density_grid(0)
    bf, mean = synth.bitfield_from_grid_numpy(grid)
    o, d, img, poses = synth.ray_batch(4096, seed=1)
    return dict(grid=grid, bitfield=bf, mean=mean, rays_o=o, rays_d=d, img_ids=img, poses=poses,
                metadata=synth.metadata_for(poses.shape[0]))
