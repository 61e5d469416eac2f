import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + '.npz'))
    out = {}
    for k in z.files:
        a = z[k]
        out[k] = torch.from_numpy(a) if a.ndim > 0 else a.item()
    return out


def mlp_of(g):
    return {k[4:]: v for k, v in g.items() if k.startswith('mlp.')}


@pytest.fixture(scope='session')
def golden():
    cache = {}
    def get(name):
        if name not in cache:
            cache[name] = load_golden(name)
        return cache[name]
    return get
