import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "gpu_new: needs a CUDA device; verified on the CPU emulation of the kernels "
                                       "(tests/test_emu_engine.py) but not yet run on a GPU - select with -m 'gpu or gpu_new'")


def _have_gpu():
    d = "/proc/driver/nvidia/gpus"
    return os.path.isdir(d) and bool(os.listdir(d))


def pytest_collection_modifyitems(config, items):
    # `-m "not gpu"` (the CPU tier) also selects the gpu_new tests: skip them where there is no device
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="gpu_new test and no CUDA device here (its CPU twin is in tests/test_emu_engine.py)")
    for it in items:
        if it.get_closest_marker("gpu_new"):
            it.add_marker(skip)


@pytest.fixture(scope="session")
def root():
    return ROOT
