"""The tracking adapters of include/openvslam_b200/adapters.hpp (adapters::search_local_landmarks and
match::projection::match_current_and_last_frames on data::frame) compile against the stand-in reference headers of tests/cpp/standin;
on a GPU box tests/cpp/test_tracking_search.cpp runs them against the class layer."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# linked into a temporary directory: the source tree may be read-only
def _build(out_dir):
    from openvslam_b200 import build
    libdir = os.path.dirname(build.build())
    exe = str(out_dir / "test_tracking_search")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "cpp", "standin"),
                           os.path.join(ROOT, "tests", "cpp", "test_tracking_search.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir,
                           "-o", exe])
    return exe


def test_tracking_adapters_compile_with_the_reference_signatures(tmp_path):
    exe = _build(tmp_path)
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_tracking_adapters_run")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr


@pytest.mark.gpu
def test_tracking_adapters_run(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "tracking search ok" in r.stdout, r.stdout + r.stderr
