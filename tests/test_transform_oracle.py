"""CPU checks of the transform optimiser's oracle (oracle/sim3_oracle.c) and of the kernel's FP64 arithmetic
(openvslam_b200/csrc/sim3_math.cuh) compiled for the host: the Sim3 exponential against scipy's expm, the analytic Jacobians
against central differences, the converged Sim3 against scipy's least_squares, and one Levenberg iteration against the numpy
restatement of tests/sim3_problems.py."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest
from scipy.linalg import expm
from scipy.optimize import least_squares

import sim3_problems as sp

HERE = os.path.dirname(os.path.abspath(__file__))
VALUES = [0.0, 1e-9, 1e-6, 1e-3, 0.7, 2.5]


@pytest.fixture(scope="module")
def s3(oracle):
    """the transform optimiser's oracle (oracle/sim3.py); `oracle` builds liboracle.so"""
    from oracle import sim3
    return sim3


def _cam(s3, model):
    return s3.camera(**sp.CAMS[model])


@pytest.mark.parametrize("theta,sigma", list(itertools.product(VALUES, VALUES)))
def test_sim3_exp_equals_expm(s3, theta, sigma):
    rng = np.random.default_rng(int(1e3 * theta) + 7 * int(1e3 * sigma))
    for _ in range(4):
        axis = rng.normal(size=3)
        u = np.concatenate([axis / np.linalg.norm(axis) * theta, rng.normal(size=3), [sigma]])
        S = s3.sim3_exp(u)
        ref = expm(sp.generator(u))
        assert np.abs(sp.to4(S) - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
        assert abs(S[12] - np.exp(sigma)) <= 1e-15 * np.exp(sigma)
        R = S[:9].reshape(3, 3)
        assert np.abs(R @ R.T - np.eye(3)).max() <= 1e-14


def test_sim3_oplus_fixed_scale_keeps_s(s3):
    rng = np.random.default_rng(3)
    S = s3.sim3_exp(np.concatenate([rng.normal(size=6) * 0.3, [0.4]]))
    for _ in range(20):
        u = rng.normal(size=7) * 0.1
        out = s3.sim3_oplus(S, u, True)
        assert out[12] == S[12]
        ref = sp.expm_oplus(S, u, True)
        assert np.abs(out - ref).max() <= 1e-13
        assert np.abs(s3.sim3_oplus(S, u, False) - sp.expm_oplus(S, u, False)).max() <= 1e-13


@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
@pytest.mark.parametrize("fix_scale", [False, True])
@pytest.mark.parametrize("forward", [True, False])
def test_edge_jacobians_match_central_differences(s3, model, fix_scale, forward):
    """J is d e(exp(xi) S) / d xi at 0 in both scale modes: fix_scale only zeroes update[6] inside oplus (the sigma column stays)"""
    p = sp.problem(30, model=model, fix_scale=fix_scale, wrong=0.0, seed=5)
    cam = _cam(s3, model)
    pc1, pc2 = sp.camera_points(p)
    S = p["S0"]
    h = 1e-6
    for i in range(0, 30, 3):
        pc, obs = (pc2[i], p["obs_xy_1"][i]) if forward else (pc1[i], p["obs_xy_2"][i])
        e, J = s3.sim3_edge(cam, S, pc, obs.astype(np.float64), forward)
        num = np.zeros((2, 7))
        for k in range(7):
            d = np.zeros(7); d[k] = h
            ep = s3.sim3_edge(cam, s3.sim3_oplus(S, d, False), pc, obs.astype(np.float64), forward)[0]
            em = s3.sim3_edge(cam, s3.sim3_oplus(S, -d, False), pc, obs.astype(np.float64), forward)[0]
            num[:, k] = (ep - em) / (2 * h)
        assert np.abs(num - J).max() <= 1e-6 * np.abs(J).max(), (i, num, J)
        # and the numpy restatement's Jacobian is the same matrix
        rows = sp.residuals(p, S, True)
        Jn = rows[2][i] if forward else rows[3][i]
        assert np.abs(Jn - J).max() <= 1e-9 * np.abs(J).max()


@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
def test_converged_sim3_equals_least_squares(s3, model):
    """outlier-free, Huber inactive (chi_sq = 1e6), free scale: the fixed point is scipy's least-squares solution"""
    p = sp.problem(150, model=model, wrong=0.0, noise=0.5, seed=9)
    cam = _cam(s3, model)
    n, S, flags, st = s3.transform_optimize(cam, cam, *sp.args(p), fix_scale=False, chi_sq=1e6)
    assert n == 150 and flags.all()
    w1, w2 = np.sqrt(p["inv_sigma_sq_1"].astype(np.float64)), np.sqrt(p["inv_sigma_sq_2"].astype(np.float64))

    def f(xi):
        e12, e21 = sp.residuals(p, sp.expm_oplus(p["S0"], xi, False))
        return np.concatenate([(e12 * w1[:, None]).ravel(), (e21 * w2[:, None]).ravel()])
    r = least_squares(f, np.zeros(7), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    S_ls = sp.expm_oplus(p["S0"], r.x, False)
    assert np.abs(S - S_ls).max() <= 1e-6, np.abs(S - S_ls).max()
    assert abs(S[12] - p["S_true"][12]) < 1e-2


@pytest.mark.parametrize("model,fix_scale", [("perspective", False), ("perspective", True), ("equirectangular", False)])
@pytest.mark.parametrize("n", [10, 60, 400])
def test_one_iteration_equals_numpy_reference(s3, model, fix_scale, n):
    p = sp.problem(n, model=model, fix_scale=fix_scale, wrong=0.0 if n == 10 else 0.15, perturb=(0.004, 0.02, 0.01), seed=n)
    cam = _cam(s3, model)
    ninl, S, flags, st = s3.transform_optimize(cam, cam, *sp.args(p), fix_scale=fix_scale, num_first_iter=1, num_iter=0)
    assert ninl >= 10, ninl
    S_ref, trials, lam0 = sp.lm_iteration(p, p["S0"], float(np.float32(np.sqrt(np.float32(10.0)))))
    assert st["num_trials"] == trials and st["round_iterations"] == [1, 0]
    assert st["lambda_init"][0] == pytest.approx(lam0, rel=1e-10)
    assert sp.step_error(S, S_ref, p["S0"]) <= 1e-10
    if fix_scale:
        assert S[12] == p["S0"][12]


def test_early_exit_leaves_the_sim3(s3):
    p = sp.problem(25, num_good=9, noise=0.3, seed=4)
    cam = _cam(s3, "perspective")
    n, S, flags, st = s3.transform_optimize(cam, cam, *sp.args(p), fix_scale=False)
    assert n == 0 and np.array_equal(S, p["S0"]) and flags.sum() == 9 and st["num_rounds"] == 1
    assert not flags[p["bad"]].any()


# ------------------------------------------------------------------ the kernel's math header, host-compiled
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sim3check") / "libsim3check.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "sim3check", "sim3check.cpp"), "-lm"])
    return C.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
def test_math_header_equals_oracle(s3, shim, model):
    rng = np.random.default_rng(12)
    cam = _cam(s3, model)
    for theta, sigma in itertools.product(VALUES, VALUES):
        axis = rng.normal(size=3)
        u = np.concatenate([axis / np.linalg.norm(axis) * theta, rng.normal(size=3), [sigma]])
        out = np.zeros(13)
        shim.sc_sim3_exp(_ptr(u), _ptr(out))
        assert np.array_equal(out, s3.sim3_exp(u))
    p = sp.problem(40, model=model, seed=13)
    pc1, pc2 = sp.camera_points(p)
    for fix in (0, 1):
        for i in range(40):
            u = rng.normal(size=7) * 0.05
            out = np.zeros(13)
            shim.sc_sim3_oplus(_ptr(p["S0"]), _ptr(u), fix, _ptr(out))
            assert np.array_equal(out, s3.sim3_oplus(p["S0"], u, fix))
    for forward in (True, False):
        fn = shim.sc_edge_forward if forward else shim.sc_edge_backward
        for i in range(40):
            pc = np.ascontiguousarray(pc2[i] if forward else pc1[i])
            obs = np.asarray(p["obs_xy_1"][i] if forward else p["obs_xy_2"][i], np.float64)
            e = np.zeros(2); J = np.zeros(14)
            fn(C.byref(cam), _ptr(p["S0"]), _ptr(pc), _ptr(obs), _ptr(e), _ptr(J))
            oe, oJ = s3.sim3_edge(cam, p["S0"], pc, obs, forward)
            assert np.array_equal(e, oe) and np.array_equal(J.reshape(2, 7), oJ)


def test_math_header_solve7(shim):
    rng = np.random.default_rng(14)
    for _ in range(50):
        A = rng.normal(size=(12, 7))
        H = A.T @ A
        b = rng.normal(size=7)
        lam = 10.0 ** rng.uniform(-6, 1)
        packed = np.array([H[i, j] for i in range(7) for j in range(i, 7)])
        x = np.zeros(7)
        assert shim.sc_solve7(_ptr(packed), C.c_double(lam), _ptr(b), _ptr(x)) == 1
        ref = np.linalg.solve(H + lam * np.eye(7), b)
        assert np.abs(x - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())
    neg = np.zeros(28); neg[0] = -1.0
    assert shim.sc_solve7(_ptr(neg), C.c_double(0.0), _ptr(np.zeros(7)), _ptr(np.zeros(7))) == 0


def test_class_layer_program_compiles_and_fails_loudly_without_gpu(tmp_path):
    """tests/cpp/test_transform_optimizer.cpp links the class layer; without a GPU it must stop with OVS_ERR_NO_DEVICE (exit 2)"""
    from openvslam_b200 import build
    import torch
    root = os.path.dirname(HERE)
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_transform_optimizer")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), os.path.join(HERE, "cpp", "test_transform_optimizer.cpp"),
                           "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_transform_optimizer_gpu.py")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
