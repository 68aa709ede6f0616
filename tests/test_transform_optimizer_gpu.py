"""optimize::transform_optimizer on the GPU (k_sim3_optimize, one launch per call) against the oracle, the numpy Levenberg
restatement of tests/sim3_problems.py and ground truth.  The kernel walks the pairs with a stride of 8 CTAs x 256 threads =
2048 pairs; the step cases sit around that stride."""
import os
import subprocess
import types

import numpy as np
import pytest

import sim3_problems as sp

pytestmark = pytest.mark.gpu

STRIDE = 2048
TOL_STEP = 1e-10
DELTA = float(np.float32(np.sqrt(np.float32(10.0))))
CONFIGS = [("perspective", False), ("perspective", True), ("equirectangular", False)]


@pytest.fixture(scope="module")
def s3(oracle):
    """the transform optimiser's oracle (oracle/sim3.py); `oracle` builds liboracle.so"""
    from oracle import sim3
    return sim3


def _run(s3, p, fix_scale, num_first_iter=5, num_iter=10, opt=None):
    from openvslam_b200 import optimize
    cam = optimize.camera(**p["cam"])
    own = opt is None
    opt = opt or optimize.transform_optimizer(fix_scale, num_iter, num_first_iter)
    g = opt.optimize(cam, cam, *sp.args(p))
    if own:
        opt.close()
    ocam = s3.camera(**p["cam"])
    o = s3.transform_optimize(ocam, ocam, *sp.args(p), fix_scale=fix_scale, num_first_iter=num_first_iter, num_iter=num_iter)
    return g, o


@pytest.mark.parametrize("n", [40, 300, 2500])
@pytest.mark.parametrize("model,fix_scale", CONFIGS)
def test_converged_equals_oracle(s3, model, fix_scale, n):
    p = sp.problem(n, model=model, fix_scale=fix_scale, seed=100 + n)
    (ninl, S, flags, st), (oninl, oS, oflags, ost) = _run(s3, p, fix_scale)
    assert ninl == oninl and ninl >= 0.7 * n
    assert np.array_equal(flags, oflags)
    assert not flags[p["bad"]].any()
    # Once a round has converged, whether a trial is accepted (and so the iteration and trial counts) turns on chi2
    # differences at rounding level, where the device's reduction tree and the oracle's loop differ; the counts are compared
    # exactly in test_one_levenberg_step, where they are determined.
    print("counts %s n=%d: device %s / %d trials, oracle %s / %d trials" % (model, n, st["round_iterations"], st["num_trials"],
                                                                          ost["round_iterations"], ost["num_trials"]))
    assert st["num_rounds"] == ost["num_rounds"] == 2
    for r in range(2):
        assert st["lambda_init"][r] == pytest.approx(ost["lambda_init"][r], rel=1e-10)
    assert np.abs(S - oS).max() <= 1e-8
    assert st["final_chi2"] == pytest.approx(ost["final_chi2"], rel=1e-8)
    assert np.abs(S - p["S_true"]).max() < 0.05
    if fix_scale:
        assert S[12] == p["S0"][12]


@pytest.mark.parametrize("n", [10, STRIDE - 1, STRIDE, STRIDE + 1, 2 * STRIDE + 1])
@pytest.mark.parametrize("model,fix_scale", CONFIGS)
def test_one_levenberg_step(s3, model, fix_scale, n):
    p = sp.problem(n, model=model, fix_scale=fix_scale, wrong=0.0 if n == 10 else 0.15, perturb=(0.004, 0.02, 0.01), seed=n)
    (ninl, S, flags, st), (oninl, oS, oflags, ost) = _run(s3, p, fix_scale, 1, 0)
    assert ninl == oninl >= 10 and np.array_equal(flags, oflags)
    assert st["num_trials"] == ost["num_trials"] and st["round_iterations"] == [1, 0]
    assert st["lambda_init"][0] == pytest.approx(ost["lambda_init"][0], rel=1e-10)
    S_ref, trials, lam0 = sp.lm_iteration(p, p["S0"], DELTA)
    assert st["num_trials"] == trials
    assert sp.step_error(S, oS, p["S0"]) <= TOL_STEP
    assert sp.step_error(S, S_ref, p["S0"]) <= TOL_STEP
    if fix_scale:
        assert S[12] == p["S0"][12]


def test_early_exit_with_nine_good_pairs(s3):
    p = sp.problem(25, num_good=9, noise=0.3, seed=4)
    (ninl, S, flags, st), (oninl, oS, oflags, ost) = _run(s3, p, False)
    assert ninl == oninl == 0
    assert np.array_equal(S, p["S0"]) and np.array_equal(oS, p["S0"])
    assert np.array_equal(flags, oflags) and flags.sum() == 9
    assert st["num_rounds"] == ost["num_rounds"] == 1


def test_no_pairs_returns_zero_without_a_launch():
    from openvslam_b200 import optimize, _lib
    p = sp.problem(20, seed=2)
    for k in ("pos_w_1", "obs_xy_1", "inv_sigma_sq_1", "pos_w_2", "obs_xy_2", "inv_sigma_sq_2"):
        p[k] = p[k][:0]
    opt = optimize.transform_optimizer(False)
    before = _lib.launch_count()
    ninl, S, flags, st = opt.optimize(optimize.camera(**p["cam"]), optimize.camera(**p["cam"]), *sp.args(p))
    assert ninl == 0 and np.array_equal(S, p["S0"]) and len(flags) == 0 and _lib.launch_count() == before
    bad = p["S0"].copy(); bad[12] = 0.0
    with pytest.raises(_lib.OvsError):
        opt.optimize(optimize.camera(**p["cam"]), optimize.camera(**p["cam"]), *sp.args(p)[:-1], bad)
    opt.close()


def test_repeated_calls_are_bit_identical(s3):
    from openvslam_b200 import optimize
    p = sp.problem(3000, model="equirectangular", seed=21)
    opt = optimize.transform_optimizer(False)
    cam = optimize.camera(**p["cam"])
    a = opt.optimize(cam, cam, *sp.args(p))
    b = opt.optimize(cam, cam, *sp.args(p))
    opt.close()
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    sa, sb = dict(a[3]), dict(b[3])
    sa.pop("device_us"); sb.pop("device_us")
    assert sa == sb


def test_invalidates_a_prepared_local_ba_on_the_same_handle():
    from openvslam_b200 import optimize, synth, _lib
    q = synth.ba_problem(6, 2, 300, model="equirectangular", seed=6)
    prep = optimize.prepared_local_ba(optimize.camera(**q["cam"]), True, q["poses"], q["fixed"], q["points"], q["obs_kf"], q["obs_lm"],
                                      q["obs_xy"], None, q["inv_sigma_sq"])
    prep.run()
    p = sp.problem(100, seed=8)
    view = types.SimpleNamespace(_h=prep._h, fix_scale_=False, num_iter_=10, num_first_iter_=5)
    ninl, S, flags, st = optimize.transform_optimizer.optimize(view, optimize.camera(**p["cam"]), optimize.camera(**p["cam"]), *sp.args(p))
    assert ninl > 70
    with pytest.raises(_lib.OvsError) as e:
        prep.run()
    assert e.value.code == -1   # OVS_ERR_INVALID_ARG
    prep.close()


def test_class_layer_against_ground_truth(tmp_path):
    from openvslam_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_transform_optimizer")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "test_transform_optimizer.cpp"), "-L", libdir, "-lovs_b200",
                           "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "transform optimizer ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("n", [100, 1000])
def test_device_time(n):
    """device_us over repeated calls after warm-up (reported, not asserted beyond being measured)"""
    from openvslam_b200 import optimize
    p = sp.problem(n, seed=30 + n)
    opt = optimize.transform_optimizer(False)
    cam = optimize.camera(**p["cam"])
    for _ in range(5):
        opt.optimize(cam, cam, *sp.args(p))
    us = [opt.optimize(cam, cam, *sp.args(p))[3]["device_us"] for _ in range(50)]
    opt.close()
    print("transform_optimizer n=%d device_us median %.1f min %.1f max %.1f" % (n, np.median(us), min(us), max(us)))
    assert all(u > 0 for u in us)
