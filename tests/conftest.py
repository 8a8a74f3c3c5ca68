import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; select with -m gpu)')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden():
    def load(name):
        return dict(np.load(os.path.join(GOLDEN, name + '.npz')))
    return load


@pytest.fixture(scope='session', autouse=True)
def _built_lib():
    """Build libdt_b200.so once if it is missing (nvcc cross-compiles on CPU)."""
    from detectandtrack_b200 import build, _lib
    if not os.path.exists(_lib.LIB_PATH):
        build.build_lib()
