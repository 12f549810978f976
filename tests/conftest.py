import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'flash-fft-conv_b200'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs an H100 (sm_90) GPU')


@pytest.fixture(scope='session')
def golden_dir():
    return os.path.join(ROOT, 'tests', 'golden')
