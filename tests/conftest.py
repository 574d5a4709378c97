import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def rel_max(a, b):
    """max|a-b| / max|b|: the parity metric of BASELINE.md (pure element-wise relative error is
    meaningless near the 1e-8 log floor and for coefficients near zero)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def noise(seed, n):
    return (0.1 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def tones(seed, n, sr):
    t = np.arange(n) / sr
    x = 0.3 * (np.sin(2 * np.pi * 220 * t) + np.sin(2 * np.pi * 880 * t) + np.sin(2 * np.pi * 3520 * t))
    return (x + 0.01 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


@pytest.fixture(scope="session")
def golden():
    def load(name):
        return np.load(os.path.join(GOLDEN, name))
    return load


@pytest.fixture(scope="session")
def ref_lib():
    from oracle import ref_lib as R
    if not R.available():
        pytest.skip("oracle/_ref/libaudioflux_ref.so not built (make -C oracle REF=<audioFlux tree>)")
    return R.get_ref_lib()


@pytest.fixture(scope="session")
def product_lib():
    from audioflux_b200 import lib as L
    try:
        return L.get_lib()
    except L.LibraryNotBuilt:
        import __graft_entry__ as g
        g.build()
        return L.get_lib()


@pytest.fixture(scope="session")
def cuda_device(product_lib):
    if product_lib.afb200_deviceCount() <= 0:
        pytest.fail("no CUDA device visible to libaudioflux_b200 (gpu-marked test on a CPU box?)")
    return 0
