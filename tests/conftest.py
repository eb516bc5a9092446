import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    import torch
    torch.set_num_threads(min(8, os.cpu_count() or 1))      # the CPU oracle does not scale to 100+ threads on tiny GEMMs
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: pytest -m gpu)')


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


class Golden:
    """Read access to a tests/golden/*.npz fixture (arrays + JSON-encoded metadata)."""

    def __init__(self, name):
        self.z = np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)

    def __getitem__(self, k):
        return self.z[k]

    def __contains__(self, k):
        return k in self.z.files

    def js(self, k):
        return json.loads(str(self.z[k]))

    def sub(self, prefix):
        """dict of arrays under ``prefix`` with the prefix stripped."""
        return {k[len(prefix):]: self.z[k] for k in self.z.files if k.startswith(prefix)}


@pytest.fixture
def golden():
    return Golden
