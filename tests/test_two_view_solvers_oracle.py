"""CPU checks of the homography / fundamental-matrix RANSAC solvers' oracle (oracle/two_view_solver_oracle.c) and of the kernels'
arithmetic (openvslam_b200/csrc/two_view_math.cuh) compiled for the host: the normalisation against a float32 numpy restatement bit
for bit, the DLT and the eight-point F against numpy SVDs (tests/two_view_problems.py), the truth, cv2.findHomography and
cv2.findFundamentalMat, every hypothesis's flags, count and score against a numpy check_inliers, the NaN rules, and the header
against the oracle bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import two_view_problems as tp

HERE = os.path.dirname(os.path.abspath(__file__))
MODELS = ["H", "F"]
IDENTITY_T4 = np.array([0.0, 0.0, 1.0, 1.0], np.float32)


@pytest.fixture(scope="module")
def tv(oracle):
    """the solvers' oracle (oracle/two_view_solver.py); `oracle` builds liboracle.so"""
    from oracle import two_view_solver
    return two_view_solver


def _close_up_to_sign(a, b, tol):
    return min(np.abs(a - b).max(), np.abs(a + b).max()) <= tol


def _unit(M):
    return M / np.linalg.norm(M)


@pytest.mark.parametrize("n", [1, 7, 100, 2000, 4000])
def test_normalize_equals_float32_numpy_bit_for_bit(tv, n):
    p = tp.problem(max(n // 2, 8), wrong=0.0, seed=n, n1=n, n2=n) if n >= 8 else None
    xy = p["keypts_1"] if p else np.random.default_rng(n).uniform(0, 640, (n, 2)).astype(np.float32)
    norm, T4 = tv.normalize(xy)
    ref, rT4 = tp.normalize(xy)
    assert np.array_equal(norm, ref, equal_nan=True) and np.array_equal(T4, rT4, equal_nan=True)   # n = 1: a zero deviation
    # over all keypoints, not only the matched ones
    if p:
        sub, sT4 = tp.normalize(xy[p["matches_12"][:, 0]])
        assert not np.array_equal(sT4, T4)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("n", [8, 9, 30, 300, 1000])
def test_minimal_solve_equals_numpy_svd(tv, model, n):
    """in normalised coordinates (identity T) within 1e-9, or 1e-15 kappa(A)^2 for a badly conditioned set (the Jacobi works on
    A^T A, which squares A's condition number); the denormalisation is T2inv (H) or T2^T (F) times it times T1"""
    for seed in range(8):
        p = tp.problem(n, scene="planar" if model == "H" else "general", wrong=0.0, noise=0.5, seed=13 * n + seed)
        q1, T1 = tp.normalize(p["keypts_1"]); q2, T2 = tp.normalize(p["keypts_2"])
        mt = p["matches_12"]
        Mn = tv.compute(model, q1, q2, mt, IDENTITY_T4, IDENTITY_T4)
        ref = tp.solve_normalised(model, q1[mt[:, 0]], q2[mt[:, 1]])
        S = np.linalg.svd(tp.design(model, q1[mt[:, 0]], q2[mt[:, 1]]), compute_uv=False)
        tol = max(1e-9, 1e-15 * (S[0] / S[7]) ** 2)
        assert _close_up_to_sign(Mn, ref, tol), (seed, np.abs(Mn - ref).max(), tol)
        M = tv.compute(model, q1, q2, mt, T1, T2)
        D = tp.denormalise(model, Mn, T1, T2)
        assert np.abs(M - D).max() <= 1e-12 * np.abs(D).max(), seed
        if model == "F":
            assert np.linalg.svd(M, compute_uv=False)[2] <= 1e-12 * np.abs(M).max()


@pytest.mark.parametrize("n", [8, 50, 500])
def test_noise_free_models_are_the_truth_and_agree_with_cv2(tv, n):
    cv2 = pytest.importorskip("cv2")
    for seed in range(5):
        for model, scene in (("H", "planar"), ("F", "general")):
            p = tp.problem(n, scene=scene, wrong=0.0, seed=5 * n + seed)
            q1, T1 = tp.normalize(p["keypts_1"]); q2, T2 = tp.normalize(p["keypts_2"])
            mt = p["matches_12"]
            M = tv.compute(model, q1, q2, mt, T1, T2)
            truth = p["H_true"] if model == "H" else p["F_true"]
            # float32 keypoints (about 3e-5 px of rounding) bound the agreement
            assert _close_up_to_sign(_unit(M), _unit(truth), 1e-5), (model, seed)
            x1, x2 = p["keypts_1"][mt[:, 0]].astype(np.float64), p["keypts_2"][mt[:, 1]].astype(np.float64)
            if model == "H":
                ref, _ = cv2.findHomography(x1, x2, 0)
            else:
                ref, _ = cv2.findFundamentalMat(x1, x2, cv2.FM_8POINT)
                assert np.linalg.matrix_rank(M, tol=1e-10 * np.abs(M).max()) == 2
            assert _close_up_to_sign(_unit(M), _unit(ref), 1e-5), (model, seed)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("noise", [0.0, 1.0])
def test_every_hypothesis_equals_numpy_check_inliers(tv, model, noise):
    """the oracle's sample, flags, count and score of every hypothesis against numpy, on data where no chi^2 lies within 1e-9 of
    its threshold (asserted)"""
    n, H, seed = 300, 60, 77
    p = tp.problem(n, scene="planar" if model == "H" else "general", wrong=0.3, noise=noise, seed=4)
    k1, k2, mt = p["keypts_1"], p["keypts_2"], p["matches_12"]
    r = tv.solve_ransac(model, k1, k2, mt, H, recompute=False, seed=seed)
    best, best_k, best_flags = 0.0, -1, None
    for k in range(H):
        assert list(r["hyp_idx"][k]) == tp.sample(seed, k, n)
        M = r["hyp_M"][k]
        flags, score, (c1, c2) = tp.check_inliers(model, M, k1, k2, mt)
        thr = tp.threshold(model)
        for c in (c1, c2):
            assert not (np.isfinite(c) & (np.abs(c - thr) <= 1e-9)).any(), "precondition: a chi^2 within 1e-9 of the threshold"
        cnt, oflags, oscore = tv.check_inliers(model, M, k1, k2, mt)
        assert np.array_equal(oflags, flags) and cnt == flags.sum() == r["hyp_count"][k], k
        assert oscore == r["hyp_score"][k]
        assert abs(score - oscore) <= 1e-11 * max(abs(score), 1.0) * n, k
        if best < score:
            best, best_k, best_flags = score, k, flags
    assert r["best_iter"] == best_k and np.array_equal(r["inliers"], best_flags)
    assert r["valid"] == (best_flags.sum() >= 8) and r["num_inliers"] == best_flags.sum()


@pytest.mark.parametrize("model", MODELS)
def test_recompute_and_small_cases(tv, model):
    p = tp.problem(400, scene="planar" if model == "H" else "general", wrong=0.3, noise=0.5, seed=5)
    k1, k2, mt = p["keypts_1"], p["keypts_2"], p["matches_12"]
    r0 = tv.solve_ransac(model, k1, k2, mt, 50, recompute=False, seed=1)
    r1 = tv.solve_ransac(model, k1, k2, mt, 50, recompute=True, seed=1)
    assert r1["valid"] and r1["best_iter"] == r0["best_iter"]
    q1, T1 = tp.normalize(k1); q2, T2 = tp.normalize(k2)
    inl = np.flatnonzero(r0["inliers"])
    ref = tv.compute(model, q1, q2, mt, T1, T2, idx=inl)
    assert np.array_equal(r1["M"], ref)
    flags, score, _ = tp.check_inliers(model, r1["M"], k1, k2, mt)
    assert np.array_equal(r1["inliers"], flags) and r1["num_inliers"] == flags.sum()
    assert abs(r1["best_score"] - score) <= 1e-10 * score
    # fewer than 8 matches: no hypothesis; 0 iterations: invalid
    for n, H in ((7, 50), (0, 50), (100, 0)):
        q = tp.problem(n, wrong=0.0, seed=6)
        r = tv.solve_ransac(model, q["keypts_1"], q["keypts_2"], q["matches_12"], H, seed=1)
        assert not r["valid"] and r["best_iter"] == -1 and (r["hyp_idx"] == -1).all() and not r["M"].any()


@pytest.mark.parametrize("model", MODELS)
def test_zero_deviation_view_gives_nan_and_loses(tv, model):
    """every keypoint of view 2 at one place: dev = 0, inv = inf, the normalised points NaN: every hypothesis is NaN, none wins"""
    p = tp.problem(60, wrong=0.0, seed=9)
    k2 = np.tile(np.float32([200.0, 100.0]), (len(p["keypts_2"]), 1))
    _, T4 = tv.normalize(k2)
    assert T4[2] == np.inf and T4[3] == np.inf
    r = tv.solve_ransac(model, p["keypts_1"], k2, p["matches_12"], 10, seed=3)
    assert np.isnan(r["hyp_M"]).any(axis=(1, 2)).all() or (r["hyp_score"] <= 0).all() or np.isnan(r["hyp_score"]).all()
    assert r["best_iter"] == -1 and not r["valid"]


def test_zero_determinant_makes_the_score_nan_and_the_hypothesis_lose(tv):
    """a singular H: the first direction passes for the match it maps exactly, the second has 0 / 0 and passes as NaN"""
    p = tp.problem(40, wrong=0.0, seed=10)
    k1, k2, mt = p["keypts_1"].copy(), p["keypts_2"].copy(), p["matches_12"]
    Hs = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 0.0]]) + np.outer([0.0, 0.0, 1.0], [0.0, 0.0, 1.0])
    Hs[1] = 0.0   # rank 2: maps every point to y = 0
    k2[mt[3, 1]] = [k1[mt[3, 0], 0], 0.0]
    assert np.linalg.det(Hs) == 0.0
    cnt, flags, score = tv.check_inliers("H", Hs, k1, k2, mt)
    ref, rscore, _ = tp.check_inliers("H", Hs, k1, k2, mt)
    assert flags[3] and np.isnan(score) and np.isnan(rscore) and np.array_equal(flags, ref) and cnt == ref.sum()


# ------------------------------------------------------------------ the kernels' math header, host-compiled
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("twoviewsolvercheck") / "libtwoviewsolvercheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "twoviewsolvercheck", "twoviewsolvercheck.cpp"), "-lm"])
    return C.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _shim_normalize(shim, xy):
    xy = np.ascontiguousarray(xy, np.float32)
    out = np.zeros((max(len(xy), 1), 2), np.float32); T4 = np.zeros(4, np.float32)
    shim.tvc_normalize(len(xy), _ptr(xy), _ptr(out), _ptr(T4))
    return out[:len(xy)], T4


def _shim_check(shim, model, M, k1, k2, mt):
    M = np.ascontiguousarray(M, np.float64).ravel()
    flags, score = np.zeros(max(len(mt), 1), np.uint8), C.c_double(0.0)
    cnt = shim.tvc_check_inliers(model, _ptr(M), len(mt), _ptr(k1), _ptr(k2), _ptr(mt), C.c_float(1.0), _ptr(flags), C.byref(score))
    return cnt, flags[:len(mt)].astype(bool), score.value


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("n,scene", [(150, "general"), (150, "planar"), (700, "general"), (2000, "planar")])
def test_header_equals_oracle_bit_for_bit(tv, shim, model, n, scene):
    """the normalisation, every hypothesis's model, flags, count and score, and the recompute over all inliers (sums past 256
    slots for the larger n)"""
    mi = 0 if model == "H" else 1
    p = tp.problem(n, scene=scene, wrong=0.25, noise=1.0, seed=n)
    k1, k2, mt = p["keypts_1"], p["keypts_2"], p["matches_12"]
    q1, T1 = _shim_normalize(shim, k1); q2, T2 = _shim_normalize(shim, k2)
    o1, oT1 = tv.normalize(k1); o2, oT2 = tv.normalize(k2)
    assert np.array_equal(q1, o1) and np.array_equal(T1, oT1) and np.array_equal(q2, o2) and np.array_equal(T2, oT2)
    H = 40
    r = tv.solve_ransac(model, k1, k2, mt, H, recompute=True, seed=13)
    for k in range(H):
        idx = np.array(r["hyp_idx"][k], np.int32)
        M = np.zeros(9)
        shim.tvc_compute(mi, 8, _ptr(q1), _ptr(q2), _ptr(mt), _ptr(idx), _ptr(T1), _ptr(T2), _ptr(M))
        assert np.array_equal(M, r["hyp_M"][k].ravel(), equal_nan=True), k
        cnt, _, score = _shim_check(shim, mi, M, k1, k2, mt)
        assert cnt == r["hyp_count"][k] and (score == r["hyp_score"][k] or (np.isnan(score) and np.isnan(r["hyp_score"][k])))
    assert r["valid"]
    _, flags, _ = _shim_check(shim, mi, r["hyp_M"][r["best_iter"]], k1, k2, mt)
    inl = np.flatnonzero(flags).astype(np.int32)
    if n >= 700 and (model == "F" or scene == "planar"):   # a homography fits a general scene's few matches only
        assert len(inl) > 256
    M = np.zeros(9)
    shim.tvc_compute(mi, len(inl), _ptr(q1), _ptr(q2), _ptr(mt), _ptr(inl), _ptr(T1), _ptr(T2), _ptr(M))
    assert np.array_equal(M, r["M"].ravel())
    c, flags, score = _shim_check(shim, mi, M, k1, k2, mt)
    assert c == r["num_inliers"] and np.array_equal(flags, r["inliers"]) and score == r["best_score"]


@pytest.mark.parametrize("model", MODELS)
def test_header_equals_oracle_on_degenerate_sets(tv, shim, model):
    mi = 0 if model == "H" else 1
    for kind in ("coincident", "collinear", "planar", "rotation"):
        p = tp.degenerate(kind, seed=3)
        k1, k2, mt = p["keypts_1"], p["keypts_2"], p["matches_12"]
        q1, T1 = _shim_normalize(shim, k1); q2, T2 = _shim_normalize(shim, k2)
        r = tv.solve_ransac(model, k1, k2, mt, 20, recompute=True, seed=2)
        for k in range(20):
            idx = np.array(r["hyp_idx"][k], np.int32)
            M = np.zeros(9)
            shim.tvc_compute(mi, 8, _ptr(q1), _ptr(q2), _ptr(mt), _ptr(idx), _ptr(T1), _ptr(T2), _ptr(M))
            assert np.array_equal(M, r["hyp_M"][k].ravel(), equal_nan=True), (kind, k)
            cnt, _, score = _shim_check(shim, mi, M, k1, k2, mt)
            assert cnt == r["hyp_count"][k] and np.array_equal(np.float64(score), np.float64(r["hyp_score"][k]), equal_nan=True)


def test_class_layer_program_compiles_and_fails_loudly_without_gpu(tmp_path):
    """tests/cpp/test_two_view_solvers.cpp links the class layer and the adapters; without a GPU it must stop with
    OVS_ERR_NO_DEVICE (exit 2)"""
    from openvslam_b200 import build
    import torch
    root = os.path.dirname(HERE)
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_two_view_solvers")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(HERE, "cpp", "standin"),
                           os.path.join(HERE, "cpp", "test_two_view_solvers.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_two_view_solvers_gpu.py")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
