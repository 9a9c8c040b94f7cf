import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


def pytest_collection_modifyitems(config, items):
    """Without a CUDA device the `gpu` tests are skipped (plain `pytest tests` on a CPU box stays green)."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason='needs a CUDA device (H100)')
    for it in items:
        if 'gpu' in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope='session')
def built():
    """Make sure librlca.so and the oracle are built (nvcc/gcc cross-compile without a GPU)."""
    import __graft_entry__ as g
    g.build(quiet=True)
    return True
