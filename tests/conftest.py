"""pytest config: `gpu` marker (tests needing an H100) + shared helpers."""
import glob
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


@pytest.fixture(scope='session')
def golden():
    import torch

    def merge(dst, src):
        for k, v in src.items():
            if isinstance(v, dict) and isinstance(dst.get(k), dict):
                merge(dst[k], v)
            else:
                dst[k] = v

    def load(name):
        path = os.path.join(ROOT, 'tests', 'golden', f'{name}.pt')
        if os.path.exists(path):
            return torch.load(path, weights_only=False)
        # stored as parts of < 1 MB each (tests/golden/make_golden.py `save`)
        parts = glob.glob(os.path.join(ROOT, 'tests', 'golden', f'{name}.[0-9]*.pt'))
        assert parts, f'no golden {name}'
        data = {}
        for part in sorted(parts, key=lambda p: int(p.rsplit('.', 2)[1])):
            merge(data, torch.load(part, weights_only=False))
        return data

    return load
