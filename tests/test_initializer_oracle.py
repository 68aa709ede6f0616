"""CPU tests of the map initialisers' oracle (oracle/initializer_oracle.c) against an independent numpy restatement
(tests/initializer_problems.py), and of the device arithmetic (openvslam_b200/csrc/initializer_math.cuh compiled with g++) against
the oracle bit for bit."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import initializer_problems as IP

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def OI():
    import oracle.initializer as OI
    return OI


def _random_matrices(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        U = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        V = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        d = np.sort(rng.uniform(0.2, 3.0, 3))[::-1] * (1.0 + np.array([0.3, 0.15, 0.0]))
        out.append(U @ np.diag(d) @ V.T)
    return out


def test_svd3_is_an_svd(OI):
    for A in _random_matrices(40, 1) + [IP.problem(50, scene="planar", seed=s)["R"] + 0.1 for s in range(5)]:
        U, d, V = OI.svd3(A)
        assert np.abs(U @ np.diag(d) @ V.T - A).max() <= 1e-12 * np.abs(A).max()
        assert np.abs(U.T @ U - np.eye(3)).max() <= 1e-12 and np.abs(V.T @ V - np.eye(3)).max() <= 1e-12
        assert np.allclose(d, np.linalg.svd(A)[1], rtol=1e-12, atol=0)
        Uc, dc, Vc = OI.svd3(A, third_by_cross=True)
        assert np.array_equal(Uc[:, :2], U[:, :2]) and np.allclose(Uc[:, 2], np.cross(U[:, 0], U[:, 1]), atol=0, rtol=0)


def test_decompositions_match_numpy(OI):
    cam = IP.PERSPECTIVE
    for A in _random_matrices(30, 2):
        H = IP.K @ A @ np.linalg.inv(IP.K)
        R, t, n = OI.decompose_homography(H, cam, cam)
        Rn, tn, nn = IP.decompose_homography(H, cam, cam)
        assert np.abs(R - Rn).max() <= 1e-9 and np.abs(t - tn).max() <= 1e-9 and np.abs(n - nn).max() <= 1e-9
        R, t = OI.decompose_essential(A)
        Rn, tn = IP.decompose_essential(A)
        assert np.abs(R - Rn).max() <= 1e-9 and np.abs(t - tn).max() <= 1e-9
        F = np.linalg.inv(IP.K).T @ A @ np.linalg.inv(IP.K)
        R, t = OI.decompose_fundamental(F, cam, cam)
        Rn, tn = IP.decompose_fundamental(F, cam, cam)
        assert np.abs(R - Rn).max() <= 1e-9 and np.abs(t - tn).max() <= 1e-9
    # equal singular values (a rotation): refused
    assert OI.decompose_homography(IP.K @ IP.problem(20, seed=3)["R"] @ np.linalg.inv(IP.K), cam, cam) is None


def _truth_index(R, t, R_true, t_true, tol_R=1e-6, tol_t=1e-5):
    tu = t_true / np.linalg.norm(t_true)
    return [h for h in range(len(R)) if np.abs(R[h] - R_true).max() <= tol_R and np.abs(t[h] - tu).max() <= tol_t]


@pytest.mark.parametrize("scene,camera,model", [("planar", "perspective", 1), ("general", "perspective", 2), ("general", "equirect", 3)])
def test_noise_free_truth_is_found_and_chosen(OI, scene, camera, model):
    """float32 keypoints bound the recovery at about 1e-7 (rotation) and 1e-6 (translation direction)"""
    for seed in (1, 3, 4):   # planar seeds 0 and 2 are ambiguous between the two physical H solutions
        p = IP.problem(300, scene=scene, camera=camera, seed=seed)
        o = OI.initialize(*IP.oracle_args(p))
        r = o["result"]
        assert r.model == model and r.status == 0, (r.model, r.status)
        assert r.chosen in _truth_index(o["hyp_R"], o["hyp_t"], p["R"], p["t"])
        s = 1.0 / np.linalg.norm(p["t"])
        tri = o["is_triangulated"]
        assert tri[p["matched_ref"]].mean() > 0.9
        truth = np.zeros((len(tri), 3)); truth[p["matched_ref"]] = p["p_ref"] * s
        err = np.linalg.norm(o["triangulated_pts"][tri] - truth[tri], axis=1) / np.linalg.norm(truth[tri], axis=1)
        assert err.max() <= 1e-3 and np.median(err) <= 1e-5   # the float32 keypoints, amplified by 1 / parallax


def _cases():
    yield IP.problem(300, scene="planar", seed=0)
    yield IP.problem(500, scene="planar", noise=1.0, wrong=0.3, seed=1)
    yield IP.problem(400, seed=2)
    yield IP.problem(800, noise=1.0, wrong=0.2, seed=3)
    yield IP.problem(300, camera="equirect", seed=4)
    yield IP.problem(600, camera="equirect", noise=1.0, wrong=0.3, seed=5)
    yield IP.problem(300, baseline=0.002, seed=1)
    yield IP.problem(200, scene="planar", baseline=0.05, seed=0)
    yield IP.problem(30, seed=7)


def test_check_pose_matches_numpy(OI):
    """counts, selected cosines and status against the vectorised numpy check_pose on the oracle's hypotheses; a match may be
    decided differently only within rounding of a threshold"""
    seen, total_diff = set(), 0
    for p in _cases():
        o = OI.initialize(*IP.oracle_args(p))
        r = o["result"]
        seen.add(r.status)
        rm = p["ref_matches_with_cur"]
        ri = np.nonzero(rm >= 0)[0]
        ci = rm[ri]
        args = (p["cam"], p["cam"], p["bearings_ref"][ri], p["bearings_cur"][ci], p["keypts_ref"][ri].astype(np.float64),
                p["keypts_cur"][ci].astype(np.float64))
        counts, coss, ndiff = [], [], 0
        for h in range(r.num_hypotheses):
            inl = o["reason"][h] != 7
            ok, small, pts, cos, margin = IP.check_pose(o["hyp_R"][h], o["hyp_t"][h], *args, inl, depth_is_positive=p["perspective"])
            diff = ok != (o["reason"][h] <= 1)
            assert (margin[diff] < 1e-6).all(), margin[diff]
            ndiff += int(diff.sum())
            # numpy's own count and selected cosine; a match decided differently within rounding moves the count by one each
            counts.append(int(ok.sum()))
            assert abs(counts[-1] - r.num_valid[h]) <= diff.sum(), (counts[-1], r.num_valid[h])
            coss.append(IP.kth_cos(cos[ok]))
            if not diff.any():
                assert abs(float(coss[-1]) - float(r.cos_parallax[h])) <= 2 * np.spacing(np.float32(1.0)), (coss[-1], r.cos_parallax[h])
        if r.num_hypotheses and ndiff == 0:
            # the decision from numpy's counts and cosines alone
            assert IP.choose(counts, coss) == (r.status, r.chosen)
        total_diff += ndiff
    assert seen >= {0, 3, 4, 5}
    assert total_diff <= 2   # the cases decide almost every match far from a threshold, so the comparison above is not vacuous


@pytest.fixture(scope="module")
def initializercheck(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("initializercheck") / "libinitializercheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "initializercheck", "initializercheck.cpp"), "-lm"])
    L = C.CDLL(so)
    L.ic_key.restype = C.c_uint
    L.ic_key_value.restype = C.c_float
    return L


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def test_header_bits_equal_the_oracle(OI, initializercheck):
    L = initializercheck
    for A in _random_matrices(20, 5):
        A = np.ascontiguousarray(A)
        for cross in (0, 1):
            U = np.zeros(9); d = np.zeros(3); V = np.zeros(9)
            L.ic_svd3(_vp(A), cross, _vp(U), _vp(d), _vp(V))
            Uo, do, Vo = OI.svd3(A, bool(cross))
            assert np.array_equal(U, Uo.ravel()) and np.array_equal(d, do) and np.array_equal(V, Vo.ravel())
    for p in _cases():
        o = OI.initialize(*IP.oracle_args(p))
        r = o["result"]
        c = OI.camera(p["cam"])
        for s in range(2 if p["perspective"] else 1):
            M = np.ascontiguousarray(np.array(r.solver_M[s][:]))
            R = np.zeros(72); t = np.zeros(24); n = np.zeros(24)
            if p["perspective"] and s == 0:
                ok = L.ic_decompose_homography(_vp(M), C.byref(c), C.byref(c), _vp(R), _vp(t), _vp(n))
                ref = OI.decompose_homography(M, p["cam"], p["cam"])
                assert bool(ok) == (ref is not None)
                if ok:
                    assert np.array_equal(R, ref[0].ravel()) and np.array_equal(t, ref[1].ravel()) and np.array_equal(n, ref[2].ravel())
            elif p["perspective"]:
                L.ic_decompose_fundamental(_vp(M), C.byref(c), C.byref(c), _vp(R), _vp(t))
                ref = OI.decompose_fundamental(M, p["cam"], p["cam"])
                assert np.array_equal(R[:36], ref[0].ravel()) and np.array_equal(t[:12], ref[1].ravel())
            else:
                L.ic_decompose_essential(_vp(M), _vp(R), _vp(t))
                ref = OI.decompose_essential(M)
                assert np.array_equal(R[:36], ref[0].ravel()) and np.array_equal(t[:12], ref[1].ravel())
        rm = p["ref_matches_with_cur"]
        ri = np.nonzero(rm >= 0)[0]
        ci = rm[ri]
        m = len(ri)
        b1 = np.ascontiguousarray(p["bearings_ref"][ri]); b2 = np.ascontiguousarray(p["bearings_cur"][ci])
        k1 = np.ascontiguousarray(p["keypts_ref"][ri]); k2 = np.ascontiguousarray(p["keypts_cur"][ci])
        for h in range(r.num_hypotheses):
            Rt = np.ascontiguousarray(np.concatenate([o["hyp_R"][h].ravel(), o["hyp_t"][h]]))
            code = np.zeros(m, np.int32); pts = np.zeros((m, 3)); cos = np.zeros(m, np.float32)
            L.ic_check_matches(_vp(Rt), C.byref(c), C.byref(c), m, _vp(b1), _vp(b2), _vp(k1), _vp(k2), C.c_double(4.0), int(p["perspective"]),
                               _vp(code), _vp(pts), _vp(cos))
            inl = o["reason"][h] != 7
            assert np.array_equal(code[inl], o["reason"][h][inl])
            for i in np.nonzero(inl)[0][:200]:
                oc, op, ocp = OI.check_match(o["hyp_R"][h], o["hyp_t"][h], p["cam"], p["cam"], b1[i], b2[i], k1[i], k2[i], 4.0, p["perspective"])
                assert oc == code[i] and np.array_equal(op, pts[i]) and ocp == cos[i]
        if r.num_hypotheses:
            cnt = np.ascontiguousarray(np.array(r.num_valid[:], np.int32)); cp = np.ascontiguousarray(np.array(r.cos_parallax[:], np.float32))
            best = C.c_int(0)
            st = L.ic_choose(r.num_hypotheses, _vp(cnt), _vp(cp), 50, C.c_double(math.cos(1.0 / 180.0 * math.pi)), C.byref(best))
            assert (st, best.value) == (r.status, r.chosen)


def test_order_preserving_key(initializercheck):
    L = initializercheck
    v = np.array([-1.0, -0.5, -1e-30, -0.0, 0.0, 1e-30, 0.3, 0.99998, 1.0], np.float32)
    keys = [L.ic_key(C.c_float(x)) for x in v]
    assert keys == sorted(keys) and keys[3] < keys[4]
    assert all(L.ic_key_value(k) == x for k, x in zip(keys, v))
    assert max(keys) < 0xffffffff


def test_cpp_initializer_compiles(tmp_path):
    """the class layer and the data::frame adapter compile with g++ against the stand-in headers; without a GPU the program reports
    it (exit code 2) instead of failing"""
    import torch
    from openvslam_b200 import build
    root = os.path.dirname(HERE)
    build.build()
    libdir = os.path.join(root, "openvslam_b200", "lib")
    exe = str(tmp_path / "test_initializer")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(HERE, "cpp", "standin"),
                           os.path.join(HERE, "cpp", "test_initializer.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_initializer_gpu.py")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
