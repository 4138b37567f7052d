import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib')
for p in (LIB, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    """On a machine without a CUDA device the gpu-marked tests are skipped (not errored), whatever -m says."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='needs a CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _fresh_cfg():
    from core import config as C
    C.reset_cfg()
    yield
    C.reset_cfg()
