import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; select with -m gpu)')


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device in this container')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def oracle():
    import oracle as orc
    orc.build()
    return orc


def synth_disc(h=512, w=512, seed=0, noise=0.05):
    """config-1 style image (SURVEY.md section 8d): background 0.25, centred disc 0.75, gaussian noise"""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[:h, :w]
    img = np.full((h, w, 3), 0.25)
    img[(yy - h / 2) ** 2 + (xx - w / 2) ** 2 < (0.3125 * min(h, w)) ** 2] = 0.75
    return np.clip(img + rng.normal(0, noise, img.shape), 0, 1)


def synth_regions(h, w, n_classes=3, seed=2, noise=0.05, cell=64):
    """config-2 style image: coarse Voronoi regions with class means 0.2/0.5/0.8 (+ per-channel offsets), noise"""
    rng = np.random.RandomState(seed)
    pts = rng.rand(40, 2) * [h, w]
    cls = rng.randint(0, n_classes, 40)
    gy, gx = np.mgrid[:(h + cell - 1) // cell, :(w + cell - 1) // cell] * cell + cell / 2
    near = ((gy[..., None] - pts[:, 0]) ** 2 + (gx[..., None] - pts[:, 1]) ** 2).argmin(-1)
    cl = np.kron(cls[near], np.ones((cell, cell), dtype=int))[:h, :w]
    means = np.linspace(0.2, 0.8, n_classes)
    img = means[cl][..., None] + np.array([0.0, 0.03, -0.03])
    return np.clip(img + rng.normal(0, noise, img.shape), 0, 1), cl
