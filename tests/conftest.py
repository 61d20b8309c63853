import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")
    config.addinivalue_line("markers", "multigpu: test needs >= 2 CUDA devices")


@pytest.fixture(autouse=True)
def _fresh_config():
    import torch
    from graphlearn_b200 import config
    config.reset()
    torch.manual_seed(0)            # model initialisations inside tests are reproducible (learning thresholds)
    yield
    config.reset()
