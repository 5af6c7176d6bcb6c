import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests are the parity tests proper and need a CUDA device; on a CPU-only box they are skipped (with the
    reason shown) instead of erroring, so that a plain `pytest tests` is green there too."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100): there is no CPU fallback of the product path")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def grid_ma2c():
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    return build_large_grid(agent="ma2c"), EnvParams(agent="ma2c")
