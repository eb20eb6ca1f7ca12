import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "compat")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with `-m gpu` on an H100)")


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from permuto_sdf_b200 import load_library
    lib = load_library()
    assert lib.psdf_device_ok() == 1, "libpsdf_b200.so loaded but the device is not sm_90 (H100)"
    return torch.device("cuda", 0)
