import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on the GPU machine with -m gpu)')


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


GOLDEN = os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture(scope='session')
def golden():
    from oracle import fixture

    def load(name):
        return fixture.expand(name, np.load(os.path.join(GOLDEN, name + '.npz')))
    return load


@pytest.fixture(scope='session')
def models():
    """(cfg, state_dict on CPU) per config, deterministic weights."""
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.model import create_model
    from geotransformer_b200.weights import synthetic_state_dict
    cache = {}

    def get(name):
        if name not in cache:
            cfg = make_cfg(name)
            model = create_model(cfg)
            sd = synthetic_state_dict(model, 7351)
            model.load_state_dict(sd, strict=True)
            cache[name] = (cfg, sd, model)
        return cache[name]
    return get
