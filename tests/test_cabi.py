"""The C-ABI shared library must load without a GPU and export every symbol that
include/ovs_b200.h declares; creating a handle without a GPU must fail loudly (no fallback)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from openvslam_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "ovs_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(ovs_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 15
    missing = [n for n in sorted(names) if not hasattr(lib, n)]
    assert not missing, missing


def test_version_and_error_string(lib):
    assert b"sm_90a" in lib.ovs_version()
    assert isinstance(lib.ovs_last_error(), bytes)


def test_no_cpu_fallback(lib):
    """Without a usable H100 handle creation returns OVS_ERR_NO_DEVICE; it never falls back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from openvslam_b200 import _lib
    h = C.c_void_p()
    p = _lib.OrbParams(1000, 1.2, 8, 20, 7)
    rc = lib.ovs_extractor_create(C.byref(p), None, 0, 0, C.byref(h))
    assert rc == -3 and b"no CPU fallback" in lib.ovs_last_error()
    rc = lib.ovs_matcher_create(0, C.byref(h))
    assert rc == -3


def test_product_does_not_import_oracle():
    """openvslam_b200/ must not reference oracle/ (the oracle is test infrastructure)."""
    pkg = os.path.join(ROOT, "openvslam_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(d, f)).read()
                assert "liboracle" not in src and "from oracle" not in src and "import oracle" not in src, f
                assert "orb_oracle" not in src and "match_oracle" not in src, f
