import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device")


def _have_gpu():
    if not os.path.exists("/dev/nvidiactl"):
        return False
    try:
        import ctypes

        n = ctypes.c_int(0)
        rt = ctypes.CDLL("libcudart.so.12")
        return rt.cudaGetDeviceCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return True  # let the tests report what is wrong


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a box without a GPU skips the gpu-marked tests (the library has no CPU fallback: fid_create
    returns FID_ERR_NO_DEVICE there) instead of failing them."""
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device: the hot path has no CPU fallback")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def kat():
    """Reference known-answer fixtures (tests/golden/make_golden.py)."""
    import cv2

    z = np.load(os.path.join(ROOT, "tests/golden/reference_kat.npz"))

    class Kat:
        def frame(self, name):
            """BGR8 pixels, stored losslessly as the top and bottom halves (tests/golden/frames)."""
            halves = [cv2.imread(os.path.join(ROOT, "tests/golden/frames", "%s_%s.webp" % (name, part)), cv2.IMREAD_COLOR) for part in ("top", "bottom")]
            return np.ascontiguousarray(np.vstack(halves))

        def __getitem__(self, k):
            return z[k]

    return Kat()


@pytest.fixture(scope="session")
def lib():
    """The C-ABI library, loaded through the python host mirror.  GPU tests only."""
    from fiducials_b200 import _lib

    return _lib.load()
