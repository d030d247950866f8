import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    # the fixture is stored in two parts (no file over 1 MB)
    return {k: v for i in (0, 1) for k, v in np.load(os.path.join(ROOT, "tests", "golden", f"unet_sampler_golden_part{i}.npz")).items()}


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Build (or reuse) the in-tree sm_90a library once per session; nvcc cross-compiles without a GPU."""
    from ivid_b200 import build
    build.build()
