import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: the kernels are built for sm_90a)')


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session', autouse=True)
def _built_library():
    """The CPU suite checks that the library loads; build it once if it is stale/missing
    (nvcc cross-compiles without a GPU)."""
    from cbgbench_b200 import build
    import shutil
    if build.is_stale() and (shutil.which('nvcc') or os.path.exists('/usr/local/cuda/bin/nvcc')):
        build.build()
    yield
