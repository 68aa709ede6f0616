"""CPU checks of the essential-matrix RANSAC solver's oracle (oracle/essential_solver_oracle.c) and of the kernel's arithmetic
(openvslam_b200/csrc/essential_math.cuh) compiled for the host: the eight-point E_21 against the numpy restatement of
tests/essential_problems.py (SVDs instead of the Jacobi), the truth and cv2.decomposeEssentialMat, the 9 x 9 Jacobi against
numpy's eigh, the sampler against numpy, every hypothesis's flags, count and score against a numpy check_inliers, and the header
against the oracle bit for bit."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import essential_problems as ep

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def es(oracle):
    """the solver's oracle (oracle/essential_solver.py); `oracle` builds liboracle.so"""
    from oracle import essential_solver
    return essential_solver


def _close_up_to_sign(a, b, tol):
    return min(np.abs(a - b).max(), np.abs(a + b).max()) <= tol


@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
@pytest.mark.parametrize("n", [8, 9, 30, 300, 1000])
def test_eight_point_equals_numpy(es, model, n):
    """within 1e-9; the Jacobi works on A^T A, which squares A's condition number, so a badly conditioned minimal set (sigma_1 /
    sigma_8 of A above ~3000) is held to 1e-15 kappa^2 instead (the numpy SVD works on A itself)"""
    for seed in range(10):
        p = ep.problem(n, model=model, wrong=0.0, noise=1e-3, seed=11 * n + seed)
        b1, b2 = p["bearings_1"], p["bearings_2"]
        E = es.compute_E(b1, b2)
        ref = ep.compute_E(b1, b2)
        S = np.linalg.svd(np.einsum("ni,nj->nij", b2, b1).reshape(-1, 9), compute_uv=False)
        tol = max(1e-9, 1e-15 * (S[0] / S[7]) ** 2)
        assert _close_up_to_sign(E, ref, tol), (seed, np.abs(E - ref).max(), np.abs(E + ref).max(), tol)


@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
@pytest.mark.parametrize("n", [8, 50, 500])
def test_noise_free_E_is_the_truth_and_decomposes(es, model, n):
    cv2 = pytest.importorskip("cv2")
    for seed in range(10):
        p = ep.problem(n, model=model, wrong=0.0, seed=3 * n + seed)
        E = es.compute_E(p["bearings_1"], p["bearings_2"])
        S = np.linalg.svd(E, compute_uv=False)
        assert abs(S[0] - S[1]) <= 1e-12 and S[2] <= 1e-12
        Et = p["E_true"] / np.linalg.norm(p["E_true"]) * np.linalg.norm(E)
        assert _close_up_to_sign(E, Et, 1e-9), seed
        R1, R2, t = cv2.decomposeEssentialMat(E)
        assert min(np.abs(R1 - p["R"]).max(), np.abs(R2 - p["R"]).max()) <= 1e-9
        th = p["t"] / np.linalg.norm(p["t"])
        assert _close_up_to_sign(t.ravel(), th, 1e-9)


def test_jacobi9_equals_eigh(es):
    from oracle import pnp_solver
    rng = np.random.default_rng(8)
    for _ in range(100):
        A = rng.normal(size=(9, 9)); A = A + A.T
        ev, V = pnp_solver.jacobi(A)
        ref = np.linalg.eigvalsh(A)
        assert np.abs(np.sort(ev) - ref).max() <= 1e-12 * np.abs(ref).max()
        assert np.abs(A @ V - V * ev).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("seed", [0, 1, 12345, 2 ** 63 + 7, 2 ** 64 - 1])
def test_sampler_draws_8_distinct_and_equals_numpy(seed):
    from oracle import oracle  # noqa: F401  (builds liboracle.so)
    from oracle import pnp_solver
    for n in list(range(8, 40)) + [255, 4000]:
        for k in range(30):
            s = pnp_solver.ransac_sample(seed, k, n, 8)
            assert s == ep.sample(seed, k, n), (n, k)
            assert len(set(s)) == 8 and all(0 <= i < n for i in s)


CASES = [("perspective", 0.0), ("perspective", 1e-3), ("equirectangular", 1e-3)]


@pytest.mark.parametrize("model,noise", CASES)
def test_every_hypothesis_equals_numpy_check_inliers(es, model, noise):
    """the oracle's sample, flags, count and score of every hypothesis against numpy, on data where no residual lies within 1e-12
    of the threshold (asserted)"""
    n, H, seed = 300, 60, 77
    p = ep.problem(n, model=model, wrong=0.3, noise=noise, seed=4)
    b1, b2 = p["bearings_1"], p["bearings_2"]
    r = es.essential_solve_ransac(b1, b2, H, recompute=False, seed=seed)
    best, best_k = 0.0, -1
    for k in range(H):
        assert list(r["hyp_idx"][k]) == ep.sample(seed, k, n)
        E = r["hyp_E"][k]
        r2, r1 = ep.residuals(E, b1, b2)
        for rr in (r2, r1):
            assert not (np.isfinite(rr) & (np.abs(rr - ep.THR) <= 1e-12)).any(), "precondition: a residual within 1e-12 of the threshold"
        flags, score = ep.check_inliers(E, b1, b2)
        cnt, oflags, oscore = es.check_inliers(E, b1, b2)
        assert np.array_equal(oflags, flags) and cnt == flags.sum() == r["hyp_count"][k], k
        assert oscore == r["hyp_score"][k]
        # a residual near 0 carries an absolute rounding error of a few ulps of 1: hence the n * 1e-15 term
        assert abs(score - oscore) <= 1e-12 * abs(score) + n * 1e-15, k
        if best < score:
            best, best_k, best_flags = score, k, flags
    assert r["best_iter"] == best_k and np.array_equal(r["inliers"], best_flags)
    assert r["valid"] == (best_flags.sum() >= 8) and r["num_inliers"] == best_flags.sum()


def test_recompute_and_small_cases(es):
    p = ep.problem(400, wrong=0.3, noise=1e-3, seed=5)
    b1, b2 = p["bearings_1"], p["bearings_2"]
    r0 = es.essential_solve_ransac(b1, b2, 50, recompute=False, seed=1)
    r1 = es.essential_solve_ransac(b1, b2, 50, recompute=True, seed=1)
    assert r1["valid"] and r1["best_iter"] == r0["best_iter"]
    ref = ep.compute_E(b1[r0["inliers"]], b2[r0["inliers"]])
    assert _close_up_to_sign(r1["E_21"], ref, 1e-9)
    flags, score = ep.check_inliers(r1["E_21"], b1, b2)
    assert np.array_equal(r1["inliers"], flags) and r1["num_inliers"] == flags.sum()
    assert abs(r1["best_score"] - score) <= 1e-12 * score
    # fewer than 8 matches: no hypothesis; 0 iterations: invalid
    for n, H in ((7, 50), (0, 50), (100, 0)):
        q = ep.problem(n, wrong=0.0, seed=6)
        r = es.essential_solve_ransac(q["bearings_1"], q["bearings_2"], H, seed=1)
        assert not r["valid"] and r["best_iter"] == -1 and (r["hyp_idx"] == -1).all() and not r["E_21"].any()


def test_zero_norm_makes_the_score_nan_and_the_hypothesis_lose(es):
    """a match whose E b1 is zero passes both tests (!(thr < NaN)) and makes the score NaN: never best"""
    p = ep.problem(40, wrong=0.0, seed=9)
    b1, b2 = p["bearings_1"].copy(), p["bearings_2"].copy()
    # E = [e_z]x (R = I, t = e_z): E e_z = 0 and E^T e_z = 0 exactly, so r2 and r1 of the pair (e_z, e_z) are 0 / 0
    E = ep.skew([0.0, 0.0, 1.0])
    b1[5] = b2[5] = [0.0, 0.0, 1.0]
    cnt, flags, score = es.check_inliers(E, b1, b2)
    ref, _ = ep.check_inliers(E, b1, b2)
    assert flags[5] and np.isnan(score) and np.array_equal(flags, ref) and cnt == ref.sum()
    # a problem whose every hypothesis meets such a pair scores NaN throughout: no best hypothesis, invalid
    q1, q2 = np.tile([0.0, 0.0, 1.0], (20, 1)), np.tile([0.0, 0.0, 1.0], (20, 1))
    r = es.essential_solve_ransac(q1, q2, 10, seed=3)
    assert np.isnan(r["hyp_score"]).all() or (r["hyp_score"] == 0).all()
    assert r["best_iter"] == -1 and not r["valid"]


# ------------------------------------------------------------------ the kernel's math header, host-compiled
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("essentialsolvercheck") / "libessentialsolvercheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "essentialsolvercheck", "essentialsolvercheck.cpp"), "-lm"])
    return C.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def test_header_sampler_and_jacobi_equal_oracle(es, shim):
    from oracle import pnp_solver
    for seed, n, k in itertools.product([0, 5, 2 ** 64 - 1], [8, 9, 17, 4000], range(30)):
        idx = (C.c_int * 8)()
        shim.esc_sample8(C.c_uint64(seed), k, n, idx)
        assert list(idx) == pnp_solver.ransac_sample(seed, k, n, 8)
    rng = np.random.default_rng(2)
    for _ in range(20):
        A = rng.normal(size=(9, 9)); A = np.ascontiguousarray(A + A.T)
        ev, V = np.zeros(9), np.zeros(81)
        shim.esc_jacobi9(_ptr(A), _ptr(ev), _ptr(V))
        oev, oV = pnp_solver.jacobi(A)
        assert np.array_equal(ev, oev) and np.array_equal(V.reshape(9, 9), oV)


@pytest.mark.parametrize("model,n", [("perspective", 150), ("equirectangular", 150), ("perspective", 700), ("equirectangular", 2000)])
def test_header_equals_oracle_bit_for_bit(es, shim, model, n):
    """every hypothesis's E_21, flags, count and score, and the recompute over all inliers (sums past 256 slots for the larger n)"""
    p = ep.problem(n, model=model, wrong=0.25, noise=1e-3, seed=n)
    b1, b2 = p["bearings_1"], p["bearings_2"]
    H = 40
    r = es.essential_solve_ransac(b1, b2, H, recompute=True, seed=13)
    for k in range(H):
        idx = np.array(r["hyp_idx"][k], np.int32)
        E = np.zeros(9)
        shim.esc_compute_E(8, _ptr(b1), _ptr(b2), _ptr(idx), _ptr(E))
        assert np.array_equal(E, r["hyp_E"][k].ravel(), equal_nan=True), k
        flags, score = np.zeros(n, np.uint8), C.c_double(0.0)
        cnt = shim.esc_check_inliers(_ptr(E), n, _ptr(b1), _ptr(b2), _ptr(flags), C.byref(score))
        assert cnt == r["hyp_count"][k] and (score.value == r["hyp_score"][k] or (np.isnan(score.value) and np.isnan(r["hyp_score"][k])))
    # the recompute: the eight-point E on the best hypothesis's inliers, in index order; also through a pair list
    flags = np.zeros(n, np.uint8)
    score = C.c_double(0.0)
    shim.esc_check_inliers(_ptr(np.ascontiguousarray(r["hyp_E"][r["best_iter"]].ravel())), n, _ptr(b1), _ptr(b2), _ptr(flags), C.byref(score))
    inl = np.flatnonzero(flags).astype(np.int32)
    E = np.zeros(9)
    shim.esc_compute_E(len(inl), _ptr(b1), _ptr(b2), _ptr(inl), _ptr(E))
    assert np.array_equal(E, r["E_21"].ravel())
    pairs = np.ascontiguousarray(np.stack([inl, inl], 1).astype(np.int32))
    E2 = np.zeros(9)
    shim.esc_compute_E_pairs(len(inl), _ptr(b1), _ptr(b2), _ptr(pairs), _ptr(E2))
    assert np.array_equal(E2, E)
    c = shim.esc_check_inliers(_ptr(E), n, _ptr(b1), _ptr(b2), _ptr(flags), C.byref(score))
    assert c == r["num_inliers"] and np.array_equal(flags.astype(bool), r["inliers"]) and score.value == r["best_score"]


def test_header_equals_oracle_on_degenerate_sets(es, shim):
    for kind in ("coincident", "collinear", "planar", "rotation"):
        p = ep.degenerate(kind, seed=3)
        b1, b2 = p["bearings_1"], p["bearings_2"]
        r = es.essential_solve_ransac(b1, b2, 20, recompute=True, seed=2)
        for k in range(20):
            idx = np.array(r["hyp_idx"][k], np.int32)
            E = np.zeros(9)
            shim.esc_compute_E(8, _ptr(b1), _ptr(b2), _ptr(idx), _ptr(E))
            assert np.array_equal(E, r["hyp_E"][k].ravel(), equal_nan=True), (kind, k)


def test_class_layer_program_compiles_and_fails_loudly_without_gpu(tmp_path):
    """tests/cpp/test_essential_solver.cpp links the class layer and the adapters; without a GPU it must stop with
    OVS_ERR_NO_DEVICE (exit 2)"""
    from openvslam_b200 import build
    import torch
    root = os.path.dirname(HERE)
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_essential_solver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(HERE, "cpp", "standin"),
                           os.path.join(HERE, "cpp", "test_essential_solver.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_essential_solver_gpu.py")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
