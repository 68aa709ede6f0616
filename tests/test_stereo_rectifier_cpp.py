"""util::stereo_rectifier in C++: tests/cpp/test_stereo_rectifier.cpp compiles adapters.hpp (the reference's constructor from the
camera and rectify(const cv::Mat&, ...)) against the stand-in reference headers of tests/cpp/standin; on a GPU box it runs the
adapter and the class layer, and their output must equal the Python path's."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# linked into a temporary directory: the source tree may be read-only
def _build(out_dir):
    from openvslam_b200 import build
    libdir = os.path.dirname(build.build())
    exe = str(out_dir / "test_stereo_rectifier")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "cpp", "standin"),
                           os.path.join(ROOT, "tests", "cpp", "test_stereo_rectifier.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir,
                           "-o", exe])
    return exe


def test_stereo_rectifier_adapter_compiles_with_the_reference_signatures(tmp_path):
    exe = _build(tmp_path)
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_stereo_rectifier_adapter_runs")
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr   # no device: an exception, no fallback


@pytest.mark.gpu
def test_stereo_rectifier_adapter_runs(tmp_path):
    from openvslam_b200 import util
    exe = _build(tmp_path)
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0 and "stereo rectifier ok" in r.stdout, r.stdout + r.stderr
    z = {k: np.fromfile(str(tmp_path / (k + ".bin")), np.float64 if k == "rig" else np.uint8)
         for k in ("rig", "raw_l", "raw_r", "out_l", "out_r", "cls_l", "cls_r")}
    rig = z["rig"]
    cols, rows = int(rig[0]), int(rig[1])
    K_l, R_l, K_r, R_r, K_rect = [rig[2 + 9 * i: 11 + 9 * i].reshape(3, 3) for i in range(5)]
    D_l, D_r = rig[47:52], rig[52:57]
    rect = util.stereo_rectifier(cols, rows, K_rect, K_l, D_l, R_l, K_r, D_r, R_r)
    pl, pr = rect.rectify(z["raw_l"].reshape(rows, cols), z["raw_r"].reshape(rows, cols))
    for side, p in (("l", pl), ("r", pr)):
        assert np.array_equal(z["out_" + side].reshape(rows, cols), p) and np.array_equal(z["cls_" + side].reshape(rows, cols), p)
    rect.close()
