import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with `-m gpu`)')


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a box without a CUDA device skips the gpu-marked tests instead of erroring in the driver stack.
    On a CUDA box nothing is skipped: a missing libubnerf_b200.so still fails loudly (no CPU / eager fallback exists)."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='needs a CUDA device (H100): run with `-m gpu` on a GPU machine')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden_dir():
    return os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture(scope='session')
def oracle():
    """CPU oracle (test infrastructure): builds oracle/libubn_oracle.so with gcc on first use."""
    from oracle import cpu_ref
    cpu_ref.build()
    return cpu_ref
