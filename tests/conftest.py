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
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100: pytest -m gpu)')


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name))


def cases_of(npz, key='cases'):
    return json.loads(bytes(npz[key]).decode())


def seeded_batches(seed, n, shape, relu):
    """Same generator as tests/golden/make_golden.py::batches (numpy legacy RandomState: bit-stable)."""
    r = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        x = r.standard_normal(size=shape).astype(np.float32)
        if relu:
            x = np.maximum(x, 0)
        out.append(x)
    return out


@pytest.fixture(scope='session')
def oracle():
    import oracle as ora
    ora.lib()
    return ora
