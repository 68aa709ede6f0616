"""The fuse adapters of include/openvslam_b200/adapters.hpp (adapters::fuse_landmark_duplication and
match::fuse::replace_duplication on a keyframe) compile against their own keyframe and landmark types in tests/cpp/test_fuse.cpp;
on a GPU box the test runs them against a sequential restatement."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# linked into a temporary directory: the source tree may be read-only
def _build(out_dir):
    from openvslam_b200 import build
    libdir = os.path.dirname(build.build())
    exe = str(out_dir / "test_fuse")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "cpp", "standin"),
                           os.path.join(ROOT, "tests", "cpp", "test_fuse.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_fuse_adapters_compile_with_the_reference_signatures(tmp_path):
    exe = _build(tmp_path)
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_fuse_adapters_run")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr


@pytest.mark.gpu
def test_fuse_adapters_run(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "fuse ok" in r.stdout, r.stdout + r.stderr
