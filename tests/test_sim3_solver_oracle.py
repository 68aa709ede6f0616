"""CPU checks of the Sim3 RANSAC solver's oracle (oracle/sim3_solver_oracle.c) and of the kernel's arithmetic
(openvslam_b200/csrc/sim3_math.cuh) compiled for the host: Horn's solution against numpy's eigh and an SVD (Umeyama) solution,
noise-free triples against the true Sim3, the sampler against a numpy restatement, and every hypothesis's inlier count against
the numpy float64 count_inliers of tests/sim3_ransac_problems.py."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation
from scipy.stats import chi2

import sim3_problems as sp
import sim3_ransac_problems as rp

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ss(oracle):
    """the solver's oracle (oracle/sim3_solver.py); `oracle` builds liboracle.so"""
    from oracle import sim3_solver
    return sim3_solver


def _sim3(rng, scale=True):
    R = Rotation.from_rotvec(rng.normal(size=3) * 0.8).as_matrix()
    return np.concatenate([R.ravel(), rng.normal(size=3), [np.exp(rng.normal() * 0.5) if scale else 1.0]])


def _apply(S, p):
    return S[12] * p @ S[:9].reshape(3, 3).T + S[9:12]


@pytest.mark.parametrize("fix_scale", [False, True])
def test_horn_equals_eigh_and_umeyama(ss, fix_scale):
    """well-conditioned noisy triples: the oracle's Jacobi + quaternion equals numpy's eigh and the SVD solution to 1e-10"""
    rng = np.random.default_rng(1 + fix_scale)
    for _ in range(200):
        S = _sim3(rng, not fix_scale)
        p2 = rng.normal(size=(3, 3)) * 2.0 + [0, 0, 6]
        p1 = _apply(S, p2) + rng.normal(size=(3, 3)) * 0.05
        S12, S21 = ss.horn(p1, p2, fix_scale)
        for ref in (rp.horn_eigh(p1, p2, fix_scale), rp.umeyama(p1, p2, fix_scale)):
            assert np.abs(S12 - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max()), (S12, ref)
        if fix_scale:
            assert S12[12] == 1.0 and S21[12] == 1.0
        # S_21 is the inverse
        assert np.abs(_apply(S21, _apply(S12, p2)) - p2).max() <= 1e-12 * max(1.0, np.abs(p2).max())
        R = S12[:9].reshape(3, 3)
        assert np.abs(R @ R.T - np.eye(3)).max() <= 1e-14


def test_jacobi_equals_eigh(ss):
    rng = np.random.default_rng(3)
    for _ in range(100):
        A = rng.normal(size=(4, 4)); A = A + A.T
        ev, V = ss.jacobi4(A)
        ref = np.linalg.eigvalsh(A)
        assert np.abs(np.sort(ev) - ref).max() <= 1e-13 * np.abs(ref).max()
        assert np.abs(A @ V - V * ev).max() <= 1e-13 * np.abs(ref).max()
        assert np.abs(V.T @ V - np.eye(4)).max() <= 1e-14


@pytest.mark.parametrize("fix_scale", [False, True])
def test_noise_free_triples_return_the_true_sim3(ss, fix_scale):
    rng = np.random.default_rng(5 + fix_scale)
    for _ in range(200):
        S = _sim3(rng, not fix_scale)
        p2 = rng.normal(size=(3, 3)) * 2.0 + [0, 0, 6]
        S12, _ = ss.horn(_apply(S, p2), p2, fix_scale)
        assert np.abs(S12 - S).max() <= 1e-12 * max(1.0, np.abs(S).max())


def test_degenerate_triples(ss):
    """coincident points: N = 0, q = (1, 0, 0, 0), R = I and a 0 / 0 scale; collinear points: a finite rotation about the line"""
    p = np.array([[1.0, 2.0, 5.0]] * 3)
    S12, S21 = ss.horn(p, p, False)
    assert np.array_equal(S12[:9], np.eye(3).ravel()) and np.isnan(S12[12])
    S12, _ = ss.horn(p, p, True)
    assert np.array_equal(S12, np.concatenate([np.eye(3).ravel(), [0, 0, 0], [1.0]]))
    q = np.array([[0.0, 0.0, 4.0], [1.0, 0.5, 5.0], [2.0, 1.0, 6.0]])
    S12, _ = ss.horn(2.0 * q, q, False)
    assert np.all(np.isfinite(S12)) and abs(S12[12] - 2.0) < 1e-12


@pytest.mark.parametrize("seed", [0, 1, 12345, 2 ** 63 + 7, 2 ** 64 - 1])
def test_sampler_equals_numpy(ss, seed):
    for n in range(3, 41):
        for k in range(0, 60):
            t = ss.ransac_triple(seed, k, n)
            assert t == rp.triple(seed, k, n), (n, k)
            assert len(set(t)) == 3 and all(0 <= i < n for i in t)
    assert ss.splitmix64_mix(seed) == rp.mix(seed)


def test_sampler_frequencies_n5():
    """all 60 ordered triples of 5 indices are equally likely: chi2 over 60000 draws"""
    counts = {}
    for k in range(60000):
        t = tuple(rp.triple(77, k, 5))
        counts[t] = counts.get(t, 0) + 1
    assert len(counts) == 60
    obs = np.array(list(counts.values()), np.float64)
    stat = ((obs - 1000.0) ** 2 / 1000.0).sum()
    assert chi2.sf(stat, 59) > 1e-3, stat


CASES = [("perspective", False), ("perspective", True), ("equirectangular", False)]


@pytest.mark.parametrize("model,fix_scale", CASES)
def test_every_hypothesis_count_equals_numpy(ss, model, fix_scale):
    """the oracle's triple and count of every hypothesis against the numpy sampler and count_inliers, on data where no error lies
    within 1e-9 relative of its bound (asserted)"""
    p = rp.problem(150, model=model, fix_scale=fix_scale, wrong=0.3, noise3d=0.01, seed=3, behind=5 if model == "perspective" else 0)
    cam = ss.camera(**p["cam"])
    seed = 99
    r = ss.sim3_solve_ransac(cam, cam, *rp.args(p), fix_scale=fix_scale, min_num_inliers=20, max_num_iter=200, seed=seed)
    pc1, pc2 = rp.camera_points(p)
    best, best_k = 0, -1
    for k in range(200):
        t = rp.triple(seed, k, 150)
        assert list(r["hyp_idx"][k]) == t
        S = rp.horn_eigh(pc1[t], pc2[t], fix_scale)
        e1, e2, ok, b1, b2 = rp.errors(p, S)
        for e, b in ((e1, b1), (e2, b2)):
            near = ok & np.isfinite(e) & (np.abs(e - b) <= 1e-9 * b)
            assert not near.any(), "precondition: an error within 1e-9 of its bound"
        inl = rp.count_inliers(p, S)
        assert r["hyp_count"][k] == inl.sum(), k
        if inl.sum() > best:
            best, best_k, best_flags, best_S = inl.sum(), k, inl, S
    assert r["num_inliers"] == best and r["best_iter"] == best_k and r["valid"] == (best >= 20)
    assert np.array_equal(r["inliers"], best_flags)
    assert np.abs(r["sim3_12"] - best_S).max() <= 1e-10 * max(1.0, np.abs(best_S).max())
    assert best >= 0.6 * 150 and not r["inliers"][p["bad"]].any()


def test_too_few_pairs_run_no_hypothesis(ss):
    p = rp.problem(19, seed=4, wrong=0.0)
    cam = ss.camera(**p["cam"])
    r = ss.sim3_solve_ransac(cam, cam, *rp.args(p), fix_scale=False, min_num_inliers=20, max_num_iter=50, seed=1)
    assert not r["valid"] and r["best_iter"] == -1 and r["num_inliers"] == 0 and (r["hyp_idx"] == -1).all()
    assert np.array_equal(r["sim3_12"], np.concatenate([np.eye(3).ravel(), [0, 0, 0], [1.0]]))
    r = ss.sim3_solve_ransac(cam, cam, *rp.args(p), fix_scale=False, min_num_inliers=10, max_num_iter=50, seed=1)
    assert r["valid"] and r["num_inliers"] == 19


# ------------------------------------------------------------------ the kernel's math header, host-compiled
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sim3solvercheck") / "libsim3solvercheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "sim3solvercheck", "sim3solvercheck.cpp"), "-lm"])
    lib = C.CDLL(so)
    lib.ssc_splitmix64_mix.restype = C.c_uint64
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def test_header_sampler_and_jacobi_equal_oracle(ss, shim):
    for seed, n, k in itertools.product([0, 5, 2 ** 64 - 1], [3, 4, 17, 4000], range(30)):
        idx = (C.c_int * 3)()
        shim.ssc_ransac_triple(C.c_uint64(seed), k, n, idx)
        assert list(idx) == ss.ransac_triple(seed, k, n)
        assert shim.ssc_splitmix64_mix(C.c_uint64(seed + k)) == ss.splitmix64_mix(seed + k)
    rng = np.random.default_rng(8)
    for _ in range(50):
        A = rng.normal(size=(4, 4)); A = A + A.T
        a = A.ravel().copy(); V = np.zeros(16)
        shim.ssc_jacobi4(_ptr(a), _ptr(V))
        ev, oV = ss.jacobi4(A)
        assert np.array_equal(np.diag(a.reshape(4, 4)), ev) and np.array_equal(V.reshape(4, 4), oV)


@pytest.mark.parametrize("model,fix_scale", CASES)
def test_header_horn_and_counts_equal_oracle(ss, shim, model, fix_scale):
    """Horn and count_inliers of the header equal the oracle bit for bit on every hypothesis of a problem with wrong pairs,
    points behind the camera and a degenerate triple"""
    p = rp.problem(120, model=model, fix_scale=fix_scale, wrong=0.3, noise3d=0.01, seed=6, behind=4 if model == "perspective" else 0)
    cam = ss.camera(**p["cam"])
    r = ss.sim3_solve_ransac(cam, cam, *rp.args(p), fix_scale=fix_scale, min_num_inliers=20, max_num_iter=100, seed=7)
    pc1, pc2 = (np.ascontiguousarray(a) for a in rp.camera_points(p))
    s1, s2 = (np.ascontiguousarray(p[k], np.float32) for k in ("sigma_sq_1", "sigma_sq_2"))
    triples = [list(t) for t in r["hyp_idx"]] + [[0, 0, 0]]
    for k, t in enumerate(triples):
        q1, q2 = np.ascontiguousarray(pc1[t]), np.ascontiguousarray(pc2[t])
        S12 = np.zeros(13); S21 = np.zeros(13)
        shim.ssc_horn(_ptr(q1), _ptr(q2), int(fix_scale), _ptr(S12), _ptr(S21))
        oS12, oS21 = ss.horn(q1, q2, fix_scale)
        assert np.array_equal(S12, oS12, equal_nan=True) and np.array_equal(S21, oS21, equal_nan=True)
        flags = np.zeros(120, np.uint8)
        c = shim.ssc_count_inliers(C.byref(cam), C.byref(cam), _ptr(S12), _ptr(S21), 120, _ptr(pc1), _ptr(pc2), _ptr(s1), _ptr(s2), _ptr(flags))
        if k < len(r["hyp_count"]):
            assert c == r["hyp_count"][k]
        if k == r["best_iter"]:
            # the camera-frame points here come from numpy, the oracle forms its own: S_12 agrees to rounding
            assert np.array_equal(flags.astype(bool), r["inliers"]) and np.abs(S12 - r["sim3_12"]).max() <= 1e-12
    rng = np.random.default_rng(9)
    for _ in range(50):
        rot = rng.normal(size=9); tr = rng.normal(size=3); pt = rng.normal(size=3) * 3
        uv = np.zeros(2)
        ok = shim.ssc_reproject(C.byref(cam), _ptr(rot), _ptr(tr), _ptr(pt), _ptr(uv))
        ook, ouv = ss.reproject(cam, rot, tr, pt)
        assert bool(ok) == ook and (not ok or np.array_equal(uv, ouv))


def test_class_layer_program_compiles_and_fails_loudly_without_gpu(tmp_path):
    """tests/cpp/test_sim3_solver.cpp links the class layer and the adapter; without a GPU it must stop with OVS_ERR_NO_DEVICE (exit 2)"""
    from openvslam_b200 import build
    import torch
    root = os.path.dirname(HERE)
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_sim3_solver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(HERE, "cpp", "standin"),
                           os.path.join(HERE, "cpp", "test_sim3_solver.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_sim3_solver_gpu.py")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
