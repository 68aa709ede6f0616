"""The C++ class layer (include/openvslam_b200/openvslam_b200.hpp: openvslam::feature::orb_extractor,
openvslam::match::*, openvslam::optimize::*) compiles and links against libovs_b200.so with g++;
on a GPU box the resulting program runs the four classes end to end."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# the programs are linked into a temporary directory: the source tree may be read-only
def _build(out_dir):
    from openvslam_b200 import build
    so = build.build()
    libdir = os.path.dirname(so)
    exe = str(out_dir / "test_class_layer")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_class_layer.cpp"),
                           "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def _build_adapters(out_dir):
    """include/openvslam_b200/adapters.hpp -- the reference's own signatures (data::frame&, data::keyframe*, std::vector<data::landmark*>,
    cv::_InputArray) -- compiled against the stand-in reference headers of tests/cpp/standin (VERDICT r1, next #8)."""
    from openvslam_b200 import build
    so = build.build()
    libdir = os.path.dirname(so)
    exe = str(out_dir / "test_adapters")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "cpp", "standin"),
                           os.path.join(ROOT, "tests", "cpp", "test_adapters.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_adapters_compile_with_the_reference_signatures(tmp_path):
    exe = _build_adapters(tmp_path)
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_adapters_run")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr


@pytest.mark.gpu
def test_adapters_run(tmp_path):
    exe = _build_adapters(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "adapters ok" in r.stdout, r.stdout + r.stderr


def test_class_layer_compiles_and_fails_loudly_without_gpu(tmp_path):
    exe = _build(tmp_path)
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_class_layer_runs")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr   # OVS_ERR_NO_DEVICE surfaced as an exception, no fallback


@pytest.mark.gpu
def test_class_layer_runs(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "class layer ok" in r.stdout, r.stdout + r.stderr
