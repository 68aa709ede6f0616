"""CPU checks of the PnP RANSAC solver's oracle (oracle/pnp_solver_oracle.c) and of the kernel's arithmetic
(openvslam_b200/csrc/pnp_math.cuh) compiled for the host: EPnP against cv2.solvePnP(SOLVEPNP_EPNP), the truth and the numpy
restatement of tests/pnp_problems.py, the sampler against numpy, every hypothesis's count against a numpy check_inliers, the
bound's polynomial cos against math.cos, and the header against the oracle bit for bit."""
import ctypes as C
import itertools
import math
import os
import subprocess

import numpy as np
import pytest

import pnp_problems as pp

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ps(oracle):
    """the solver's oracle (oracle/pnp_solver.py); `oracle` builds liboracle.so"""
    from oracle import pnp_solver
    return pnp_solver


def _cv2_pose(p):
    cv2 = pytest.importorskip("cv2")
    b = p["bearings"]
    img = np.ascontiguousarray(b[:, :2] / b[:, 2:3])
    ok, rvec, tvec = cv2.solvePnP(p["pos_w"], img, np.eye(3), None, flags=cv2.SOLVEPNP_EPNP)
    assert ok
    return np.concatenate([cv2.Rodrigues(rvec)[0].ravel(), tvec.ravel()])


@pytest.mark.parametrize("n", [6, 10, 100, 1000])
def test_epnp_equals_cv2_and_the_truth_noise_free(ps, n):
    for seed in range(20):
        p = pp.problem(n, wrong=0.0, seed=100 * n + seed)
        pose = ps.epnp(p["bearings"], p["pos_w"])
        assert np.abs(pose - p["pose_true"]).max() <= 1e-9, (seed, pose - p["pose_true"])
        assert np.abs(pose - _cv2_pose(p)).max() <= 1e-9


@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
@pytest.mark.parametrize("n", [6, 7, 30, 300])
def test_epnp_equals_numpy_on_noisy_bearings(ps, model, n):
    for seed in range(10):
        p = pp.problem(n, model=model, wrong=0.0, noise=1e-3, seed=7 * n + seed)
        pose = ps.epnp(p["bearings"], p["pos_w"])
        ref = pp.epnp(p["bearings"], p["pos_w"])
        assert np.abs(pose - ref).max() <= 1e-9, (seed, np.abs(pose - ref).max())
        if n >= 30:
            assert np.abs(pose - p["pose_true"]).max() <= 0.05


def test_planar_failure_rates_are_reported(ps):
    """exactly planar scenes are a known weakness of EPnP: the rates are printed next to cv2's, not asserted"""
    for n in (6, 30, 300):
        ours = theirs = 0
        for seed in range(100):
            p = pp.problem(n, wrong=0.0, seed=5000 + seed, planar=True)
            ours += np.abs(ps.epnp(p["bearings"], p["pos_w"]) - p["pose_true"]).max() > 1e-6
            theirs += np.abs(_cv2_pose(p) - p["pose_true"]).max() > 1e-6
        print("planar n=%d: oracle fails %d %%, cv2 fails %d %%" % (n, ours, theirs))


@pytest.mark.parametrize("seed", [0, 1, 12345, 2 ** 63 + 7, 2 ** 64 - 1])
def test_sampler_equals_numpy(ps, seed):
    for n in range(6, 40):
        for k in range(40):
            s = ps.ransac_sample(seed, k, n)
            assert s == pp.sample(seed, k, n), (n, k)
            assert len(set(s)) == 6 and all(0 <= i < n for i in s)
    # m = 3 is the Sim3 solver's triple
    from oracle import sim3_solver
    for n, k in itertools.product([3, 4, 17, 4000], range(30)):
        assert ps.ransac_sample(seed, k, n, 3) == sim3_solver.ransac_triple(seed, k, n)


def test_jacobi_equals_eigh(ps):
    rng = np.random.default_rng(3)
    for N in (3, 12):
        for _ in range(50):
            A = rng.normal(size=(N, N)); A = A + A.T
            ev, V = ps.jacobi(A)
            ref = np.linalg.eigvalsh(A)
            assert np.abs(np.sort(ev) - ref).max() <= 1e-12 * np.abs(ref).max()
            assert np.abs(A @ V - V * ev).max() <= 1e-12 * np.abs(ref).max()


def test_max_cos_within_one_ulp_of_math_cos(ps):
    rng = np.random.default_rng(4)
    sf = np.concatenate([rng.uniform(0.0, 90.0, 20000), 1.2 ** np.arange(0, 25), [1e-6, 44.9999, 45.0, 45.0001, 89.99, 90.0]])
    sf = np.unique(sf.astype(np.float32))
    sf = sf[(sf > 0) & (sf <= 90)]
    for s in sf:
        ref = math.cos(math.pi / 180.0 * float(s))
        got = ps.max_cos(float(s))
        assert abs(got - ref) <= math.ulp(ref), (s, got, ref)


CASES = [("perspective", 0.0), ("perspective", 1e-3), ("equirectangular", 1e-3)]


@pytest.mark.parametrize("model,noise", CASES)
def test_every_hypothesis_count_equals_numpy(ps, model, noise):
    """the oracle's sample and count of every hypothesis against the numpy sampler and check_inliers, on data where no cosine
    lies within 1e-12 of its bound (asserted)"""
    n, H, seed = 200, 60, 99
    p = pp.problem(n, model=model, wrong=0.3, noise=noise, seed=3)
    r = ps.pnp_solve_ransac(*pp.args(p), min_num_inliers=10, max_num_iter=H, recompute=False, seed=seed)
    best, best_k = 0, -1
    bound = pp.max_cos(p["scale_factor"])
    for k in range(H):
        assert list(r["hyp_idx"][k]) == pp.sample(seed, k, n)
        pose = r["hyp_pose"][k]
        with np.errstate(invalid="ignore", divide="ignore"):
            cs = pp.cosines(pose, p["bearings"], p["pos_w"])
        assert not (np.isfinite(cs) & (np.abs(cs - bound) <= 1e-12)).any(), "precondition: a cosine within 1e-12 of its bound"
        inl = pp.check_inliers(pose, p)
        assert r["hyp_count"][k] == inl.sum(), k
        if inl.sum() > best:
            best, best_k, best_flags = inl.sum(), k, inl
    assert r["num_inliers"] == best and r["best_iter"] == best_k and r["valid"] == (best >= 10)
    assert np.array_equal(r["inliers"], best_flags)
    assert best >= 0.6 * n and not r["inliers"][p["bad"]].any()


def test_recompute_and_small_cases(ps):
    p = pp.problem(300, wrong=0.3, noise=1e-3, seed=5)
    r0 = ps.pnp_solve_ransac(*pp.args(p), min_num_inliers=10, max_num_iter=30, recompute=False, seed=1)
    r1 = ps.pnp_solve_ransac(*pp.args(p), min_num_inliers=10, max_num_iter=30, recompute=True, seed=1)
    assert r1["valid"] and r1["best_iter"] == r0["best_iter"]
    ref = pp.epnp(p["bearings"][r0["inliers"]], p["pos_w"][r0["inliers"]])
    assert np.abs(r1["pose_cw"] - ref).max() <= 1e-9
    assert np.array_equal(r1["inliers"], pp.check_inliers(r1["pose_cw"], p)) and r1["num_inliers"] == r1["inliers"].sum()
    # fewer than 6 or fewer than min_num_inliers correspondences: no hypothesis
    for n, m in ((5, 0), (9, 10)):
        q = pp.problem(n, wrong=0.0, seed=6)
        r = ps.pnp_solve_ransac(*pp.args(q), min_num_inliers=m, max_num_iter=30, seed=1)
        assert not r["valid"] and r["best_iter"] == -1 and (r["hyp_idx"] == -1).all()


# ------------------------------------------------------------------ the kernel's math header, host-compiled
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pnpsolvercheck") / "libpnpsolvercheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "pnpsolvercheck", "pnpsolvercheck.cpp"), "-lm"])
    lib = C.CDLL(so)
    lib.psc_max_cos.restype = C.c_double
    lib.psc_max_cos.argtypes = [C.c_float]
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def test_header_sampler_and_bound_equal_oracle(ps, shim):
    for seed, n, k in itertools.product([0, 5, 2 ** 64 - 1], [6, 7, 17, 4000], range(30)):
        idx = (C.c_int * 6)()
        shim.psc_sample6(C.c_uint64(seed), k, n, idx)
        assert list(idx) == ps.ransac_sample(seed, k, n)
    for s in np.float32(1.2) ** np.arange(0, 25, dtype=np.float32):
        if s <= 90:
            assert shim.psc_max_cos(float(s)) == ps.max_cos(float(s))


@pytest.mark.parametrize("model,n", [("perspective", 150), ("equirectangular", 150), ("perspective", 700), ("equirectangular", 2000)])
def test_header_equals_oracle_bit_for_bit(ps, shim, model, n):
    """every hypothesis's EPnP pose and count, and the recompute over all inliers (sums past 256 slots for the larger n)"""
    p = pp.problem(n, model=model, wrong=0.2, noise=1e-3, seed=n)
    b, w, s = (np.ascontiguousarray(a) for a in pp.args(p))
    r = ps.pnp_solve_ransac(b, w, s, min_num_inliers=10, max_num_iter=30, recompute=True, seed=11)
    for k in range(30):
        idx = np.array(r["hyp_idx"][k], np.int32)
        pose = np.zeros(12)
        shim.psc_epnp(6, _ptr(b), _ptr(w), _ptr(idx), _ptr(pose))
        assert np.array_equal(pose, r["hyp_pose"][k], equal_nan=True), k
        assert shim.psc_check_inliers(n, _ptr(b), _ptr(w), _ptr(s), _ptr(pose), None) == r["hyp_count"][k]
    # the recompute: EPnP on the best hypothesis's inliers, in index order
    best = np.array(r["hyp_pose"][r["best_iter"]])
    flags = np.zeros(n, np.uint8)
    shim.psc_check_inliers(n, _ptr(b), _ptr(w), _ptr(s), _ptr(best), _ptr(flags))
    inl = np.flatnonzero(flags).astype(np.int32)
    pose = np.zeros(12)
    shim.psc_epnp(len(inl), _ptr(b), _ptr(w), _ptr(inl), _ptr(pose))
    assert np.array_equal(pose, r["pose_cw"])
    c = shim.psc_check_inliers(n, _ptr(b), _ptr(w), _ptr(s), _ptr(pose), _ptr(flags))
    assert c == r["num_inliers"] and np.array_equal(flags.astype(bool), r["inliers"])


def test_header_equals_oracle_on_degenerate_sets(ps, shim):
    for kind in ("coincident", "collinear", "planar"):
        p = pp.degenerate(kind, seed=3)
        b, w, s = (np.ascontiguousarray(a) for a in pp.args(p))
        r = ps.pnp_solve_ransac(b, w, s, min_num_inliers=6, max_num_iter=20, recompute=True, seed=2)
        for k in range(20):
            idx = np.array(r["hyp_idx"][k], np.int32)
            pose = np.zeros(12)
            shim.psc_epnp(6, _ptr(b), _ptr(w), _ptr(idx), _ptr(pose))
            assert np.array_equal(pose, r["hyp_pose"][k], equal_nan=True), (kind, k)


def test_class_layer_program_compiles_and_fails_loudly_without_gpu(tmp_path):
    """tests/cpp/test_pnp_solver.cpp links the class layer and the adapter; without a GPU it must stop with OVS_ERR_NO_DEVICE (exit 2)"""
    from openvslam_b200 import build
    import torch
    root = os.path.dirname(HERE)
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_pnp_solver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(HERE, "cpp", "standin"),
                           os.path.join(HERE, "cpp", "test_pnp_solver.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_pnp_solver_gpu.py")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
