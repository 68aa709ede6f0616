import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with -m gpu)")


def _has_gpu():
    try:
        import ctypes
        from openvslam_b200 import _lib
        h = ctypes.c_void_p()
        rc = _lib.lib().ovs_matcher_create(0, ctypes.byref(h))
        if rc == 0:
            _lib.lib().ovs_matcher_destroy(h)
        return rc == 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # -m gpu tests must FAIL, not skip, if the CUDA library is unusable on a GPU box; on a box
    # without a GPU they are deselected by `-m "not gpu"`.  Nothing to do here.
    return


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "cv2_primitives.npz"))
