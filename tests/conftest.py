import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a)")
    config.addinivalue_line("markers", "slow: long-running CPU test")


@pytest.fixture(scope="session")
def smplh_np():
    from interdiff_b200 import synthetic
    return synthetic.make_smplh_model(233)
