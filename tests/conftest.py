import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an sm_90 CUDA device (H100)")


def _device_ok():
    try:
        import torch
        return torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0)
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need an sm_90 device: without one they are skipped (plain `pytest tests` on a CPU box), unless
    they were asked for explicitly with `-m gpu` -- on the GPU box a missing device must fail loudly, not skip."""
    if _device_ok() or "gpu" in (config.getoption("-m") or ""):
        return
    skip = pytest.mark.skip(reason="needs an sm_90a CUDA device (H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle_pp():
    from oracle import postproc_oracle as P

    P.build()
    return P
