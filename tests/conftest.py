import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: test needs a CUDA device (run on an H100)')


@pytest.fixture(scope='session')
def golden_dir():
    return GOLDEN


@pytest.fixture(scope='session')
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail('this test is marked gpu and needs a CUDA device (no CPU fallback exists)')
    return torch.device('cuda:0')
