import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
for p in (ROOT, GOLDEN_DIR):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def _cuda_device_count() -> int:
    """Devices the CUDA driver reports (0 when there is no driver).  Deliberately independent of
    this package's library: a box WITH a GPU must run the gpu tests and fail loudly if the
    extension is broken; only a box without any device skips them."""
    import ctypes
    try:
        cuda = ctypes.CDLL("libcuda.so.1")
    except OSError:
        return 0
    n = ctypes.c_int(0)
    if cuda.cuInit(0) != 0 or cuda.cuDeviceGetCount(ctypes.byref(n)) != 0:
        return 0
    return n.value


def pytest_collection_modifyitems(config, items):
    gpu_items = [it for it in items if it.get_closest_marker("gpu")]
    if gpu_items and _cuda_device_count() == 0:
        skip = pytest.mark.skip(reason="no CUDA device visible (gpu tests run on an H100)")
        for it in gpu_items:
            it.add_marker(skip)


def _unjson_float(x):
    return float(x) if isinstance(x, str) else x


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(GOLDEN_DIR, "golden.json")) as fh:
        return json.load(fh)


@pytest.fixture(scope="session")
def golden_arrays():
    return np.load(os.path.join(GOLDEN_DIR, "golden_arrays.npz"))


@pytest.fixture(scope="session")
def gf():
    """json float decoder: fixtures store -inf/nan as strings."""
    return _unjson_float
