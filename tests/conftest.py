import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on the GPU box)")


def _has_gpu():
    try:
        import ctypes
        cuda = ctypes.CDLL("libcuda.so.1")
        if cuda.cuInit(0) != 0:
            return False
        n = ctypes.c_int()
        return cuda.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return False


HAS_GPU = _has_gpu()


def pytest_collection_modifyitems(config, items):
    if HAS_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def fixture_gd_input(oracle):
    """The reference suite's data (Suite.scala:32-49): generateGDInput(2.0, -1.5, 10000, 42) with an
    intercept column of ones prepended."""
    import numpy as np
    x1, y = oracle.generate_gd_input(2.0, -1.5, 10000, 42)
    X = np.stack([np.ones_like(x1), x1], axis=1)
    return y, X


@pytest.fixture(scope="session")
def agd():
    import spark_agd_b200
    return spark_agd_b200


@pytest.fixture(scope="session")
def ctx(agd):
    return agd.Context(devices=[0])
