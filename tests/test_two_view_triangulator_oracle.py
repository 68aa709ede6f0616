"""CPU tests of the two-view triangulator's oracle (oracle/triangulation_oracle.c) against numpy restatements, of the device
arithmetic (openvslam_b200/csrc/triangulation_math.cuh compiled with g++) against the oracle bit for bit, and of the oracle's
create_new_landmarks against a Python loop over the oracle's matcher and triangulator."""
import collections
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import triangulation_problems as TP
from openvslam_b200 import module

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def OT(oracle):
    from oracle import triangulation
    return triangulation


def _A(b1, b2, P1, P2):
    P1 = P1.reshape(3, 4); P2 = P2.reshape(3, 4)
    return np.array([b1[0] * P1[2] - b1[2] * P1[0], b1[1] * P1[2] - b1[2] * P1[1], b2[0] * P2[2] - b2[2] * P2[0], b2[1] * P2[2] - b2[2] * P2[1]])


def _P(kf):
    return np.concatenate([kf.pose_cw[:9].reshape(3, 3), kf.pose_cw[9:, None]], 1)


def _rays(kf, i):
    return kf.pose_cw[:9].reshape(3, 3).T @ kf.bearings[i]


def _centre(kf):
    R = kf.pose_cw[:9].reshape(3, 3)
    return -(R.T @ kf.pose_cw[9:])


def _cases():
    """(kf1, kf2, pairs): perspective mono, stereo, close stereo, equirectangular, a camera looking back and a far-away camera"""
    out = [TP.pair_problem(1, 3000), TP.pair_problem(2, 3000, stereo_frac=0.5), TP.pair_problem(3, 3000, stereo_frac=0.5, spacing=0.02),
           TP.pair_problem(4, 2000, "equirectangular")]
    kf1, kf2, pairs = TP.pair_problem(5, 1500, stereo_frac=0.8)
    R = kf2.pose_cw[:9].reshape(3, 3) @ np.diag([-1.0, 1.0, -1.0])     # keyframe 2 turned around: points behind it
    back = module.keyframe(np.concatenate([R.reshape(9), -R @ _centre(kf2)]), kf2.camera, kf2.scale_factor, kf2.scale_factors,
                           kf2.level_sigma_sq, kf2.keypts["x"], kf2.keypts["y"], kf2.keypts["octave"], kf2.bearings,
                           stereo_x_right=kf2.stereo_x_right, depths=kf2.depths, true_baseline=kf2.true_baseline)
    out.append((kf1, back, pairs))
    far = module.keyframe(np.concatenate([kf2.pose_cw[:9], [1e160, 0.0, 0.0]]), kf2.camera, kf2.scale_factor, kf2.scale_factors,
                          kf2.level_sigma_sq, kf2.keypts["x"], kf2.keypts["y"], kf2.keypts["octave"], kf2.bearings)
    kf1m = module.keyframe(kf1.pose_cw, kf1.camera, kf1.scale_factor, kf1.scale_factors, kf1.level_sigma_sq, kf1.keypts["x"], kf1.keypts["y"],
                           kf1.keypts["octave"], kf1.bearings)
    out.append((kf1m, far, pairs[:300]))
    return out


def _reason_numpy(kf1, kf2, i1, i2, pos, cos_thr):
    """the reference's tests restated in numpy, given the oracle's point for the two-camera branch"""
    def stereo(kf, i):
        return kf.stereo_x_right is not None and kf.stereo_x_right[i] >= 0
    st1, st2 = stereo(kf1, i1), stereo(kf2, i2)
    r1, r2 = _rays(kf1, i1), _rays(kf2, i2)
    cos_rays = r1 @ r2 / (np.linalg.norm(r1) * np.linalg.norm(r2))

    def cs(kf, i, st):
        return math.cos(2 * math.atan2(kf.true_baseline / 2, float(kf.depths[i]))) if st else 2.0
    c1, c2 = cs(kf1, i1, st1), cs(kf2, i2, st2)
    tol = 1e-12                                  # closed form vs cos(2 atan2): a pair this close to a threshold is skipped
    if (not st1 and not st2 and 0 < cos_rays < cos_thr) or ((st1 or st2) and 0 < cos_rays < min(c1, c2)):
        if (st1 or st2) and abs(cos_rays - min(c1, c2)) < tol:
            return None
        if not np.all(np.isfinite(pos)):
            return 2
    elif st1 and c1 < c2:
        kf, i = kf1, i1
    elif st2 and c2 < c1:
        kf, i = kf2, i2
    else:
        return None if (st1 or st2) and abs(c1 - c2) < tol else 1
    for v, kf in ((0, kf1), (1, kf2)):
        if kf.camera.model == 0:
            R = kf.pose_cw[:9].reshape(3, 3)
            if not np.float32(R[2] @ pos + kf.pose_cw[11]) > 0:
                return 3 + v
    for v, (kf, i) in enumerate(((kf1, i1), (kf2, i2))):
        R = kf.pose_cw[:9].reshape(3, 3)
        pc = R @ pos + kf.pose_cw[9:]
        if kf.camera.model == 0:
            u = kf.camera.fx * pc[0] / pc[2] + kf.camera.cx; w = kf.camera.fy * pc[1] / pc[2] + kf.camera.cy
        else:
            b = pc / np.linalg.norm(pc)
            u = kf.camera.cols * (0.5 + math.atan2(b[0], b[2]) / (2 * math.pi)); w = kf.camera.rows * (0.5 + math.asin(b[1]) / math.pi)
        e2 = (u - kf.keypts["x"][i]) ** 2 + (w - kf.keypts["y"][i]) ** 2
        sig = kf.level_sigma_sq[kf.keypts["octave"][i]]
        if stereo(kf, i):
            xr = np.float32(u - kf.camera.focal_x_baseline / pc[2])
            bound, err = float(np.float32(7.81473) * sig), e2 + float((xr - kf.stereo_x_right[i]) ** 2)
        else:
            bound, err = float(np.float32(5.99146) * sig), e2
        if abs(err - bound) < 1e-9 * bound:
            return None
        if bound < err:
            return 5 + v
    d1, d2 = np.linalg.norm(pos - _centre(kf1)), np.linalg.norm(pos - _centre(kf2))
    f = np.float32(1.5) * np.float32(kf1.scale_factor)
    ro = np.float32(kf1.scale_factors[kf1.keypts["octave"][i1]]) / np.float32(kf2.scale_factors[kf2.keypts["octave"][i2]])
    if d1 == 0 or d2 == 0 or d2 / d1 * f < ro or float(ro * f) < d2 / d1:
        return 7
    return 0


def test_two_camera_solution_against_numpy_svd(OT):
    """parallax >= 1 degree: the point from the 4 x 4 Jacobi on A^T A within 1e-9 (relative) of numpy's SVD of A"""
    kf1, kf2, pairs = TP.pair_problem(11, 4000)
    v, pos, reason, branch = OT.triangulate(kf1, kf2, pairs, rays_parallax_deg_thr=1.0)
    checked = 0
    worst = 0.0
    for k in np.flatnonzero((branch == 0) & (reason != 2)):
        i1, i2 = pairs[k]
        _, _, Vt = np.linalg.svd(_A(kf1.bearings[i1], kf2.bearings[i2], _P(kf1), _P(kf2)))
        ref = Vt[3, :3] / Vt[3, 3]
        p = _point(OT, kf1, kf2, i1, i2)
        worst = max(worst, np.linalg.norm(p - ref) / np.linalg.norm(ref))
        checked += 1
    assert checked > 500 and worst < 1e-9, (checked, worst)


def test_noise_free_points_are_recovered(OT):
    rng = np.random.default_rng(12)
    scene = TP.make_scene(rng, 2000)
    kf1, p1 = TP.make_keyframe(rng, scene, np.zeros(3), TP.rot(rng, 1.0), noise_px=0.0, outlier_frac=0.0, n_distractors=0)
    kf2, p2 = TP.make_keyframe(rng, scene, np.array([0.6, 0.05, 0.1]), TP.rot(rng, 3.0), noise_px=0.0, outlier_frac=0.0, n_distractors=0)
    # exact bearings of the points (the keypoints are rounded to float)
    for kf, p in ((kf1, p1), (kf2, p2)):
        R = kf.pose_cw[:9].reshape(3, 3)
        Xc = scene["X"][p] @ R.T + kf.pose_cw[9:]
        kf.bearings[:] = Xc / np.linalg.norm(Xc, axis=1, keepdims=True)
    inv2 = {int(q): i for i, q in enumerate(p2)}
    pairs = np.array([(i, inv2[int(q)]) for i, q in enumerate(p1) if int(q) in inv2], np.int32)
    valid, pos, reason, branch = OT.triangulate(kf1, kf2, pairs)
    X = scene["X"][p1[pairs[:, 0]]]
    two = branch == 0
    assert two.sum() > 500
    # the octaves are random, so the scale test rejects some pairs: the point is checked before it
    P = np.array([_point(OT, kf1, kf2, i1, i2) for i1, i2 in pairs[two]])
    err = np.linalg.norm(P - X[two], axis=1) / np.linalg.norm(X[two], axis=1)
    assert err.max() < 1e-9 and np.array_equal(pos[two & valid], P[valid[two]])


def test_every_gate_agrees_with_numpy(OT):
    cos_thr = math.cos(1.0 / 180.0 * math.pi)
    seen = collections.Counter()
    for kf1, kf2, pairs in _cases():
        valid, pos, reason, branch = OT.triangulate(kf1, kf2, pairs)
        for k, (i1, i2) in enumerate(pairs):
            p = pos[k]
            if reason[k] not in (0, 1) and branch[k] >= 0:
                p = _point(OT, kf1, kf2, i1, i2)
            ref = _reason_numpy(kf1, kf2, i1, i2, p, cos_thr)
            if ref is None:
                continue
            assert reason[k] == ref, (k, reason[k], ref)
            st = lambda kf, i: kf.stereo_x_right is not None and kf.stereo_x_right[i] >= 0
            tag = {5: ("reproj 1", bool(st(kf1, i1))), 6: ("reproj 2", bool(st(kf2, i2)))}.get(int(reason[k]), int(reason[k]))
            seen[tag] += 1
            seen[("branch", int(branch[k]))] += 1
    for want in (0, 1, 2, 3, 4, 7, ("reproj 1", True), ("reproj 1", False), ("reproj 2", True), ("reproj 2", False),
                 ("branch", 0), ("branch", 1), ("branch", 2), ("branch", -1)):
        assert seen[want] > 0, (want, seen)


def _point(OT, kf1, kf2, i1, i2):
    """the point of a rejected pair, from the oracle with every gate opened: the same arithmetic up to the failing test"""
    import oracle.triangulation as T
    lib = T.lib()
    keep = []
    k1 = T._kf(kf1, keep); k2 = T._kf(kf2, keep)
    p = (C.c_double * 3)(); br = C.c_int(0)
    lib.otr_triangulate(C.byref(k1), C.byref(k2), int(i1), int(i2), C.c_double(math.cos(math.pi / 180.0)), p, C.byref(br))
    return np.array(list(p))


@pytest.fixture(scope="module")
def triangulationcheck(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("triangulationcheck") / "libtriangulationcheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "triangulationcheck", "triangulationcheck.cpp"), "-lm"])
    return C.CDLL(so)


def test_header_bits_equal_the_oracle(OT, triangulationcheck):
    import oracle.triangulation as T
    cos_thr = math.cos(1.0 / 180.0 * math.pi)
    for kf1, kf2, pairs in _cases():
        keep = []
        k1 = T._kf(kf1, keep); k2 = T._kf(kf2, keep)
        m = len(pairs)
        pos = np.zeros((m, 3)); reason = np.zeros(m, np.int32); branch = np.zeros(m, np.int32)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        triangulationcheck.tc_two_view_triangulate(C.byref(k1), C.byref(k2), m, vp(np.ascontiguousarray(pairs)), C.c_double(cos_thr), vp(pos),
                                                   vp(reason), vp(branch))
        valid, opos, oreason, obranch = OT.triangulate(kf1, kf2, pairs)
        assert np.array_equal(reason, oreason) and np.array_equal(branch, obranch)
        assert pos.tobytes() == opos.tobytes()


@pytest.mark.parametrize("B,check", [(1, False), (6, True), (12, False)])
def test_oracle_create_new_landmarks_is_the_sequential_loop(oracle, OT, B, check):
    kf1, nbs, E, ep = TP.neighbourhood(20 + B, 1500, B, stereo_frac=0.3)
    rec, pos = OT.create_new_landmarks(kf1, nbs, E, ep, check)
    has = kf1.has_landmark.copy()
    keys = []
    for b, n in enumerate(nbs):
        st1 = (kf1.stereo_x_right >= 0).astype(np.uint8); st2 = (n.stereo_x_right >= 0).astype(np.uint8)
        _, m = oracle.robust_match_for_triangulation(kf1.descriptors, kf1.bearings, kf1.keypts["octave"], kf1.keypts["angle"], has, st1,
                                                     kf1.bow_node, n.descriptors, n.bearings, n.keypts["angle"], n.has_landmark, st2,
                                                     n.bow_node, E[b], ep[b], kf1.scale_factors, check)
        i1 = np.flatnonzero(m >= 0)
        valid, p, _, _ = OT.triangulate(kf1, n, np.stack([i1, m[i1]], 1))
        for k in np.flatnonzero(valid):
            keys.append((b, i1[k], m[i1[k]], *p[k]))
            has[i1[k]] = 1
    ref = np.array(keys).reshape(-1, 6)
    assert len(rec) == len(ref) and len(rec) > 100
    assert np.array_equal(rec, ref[:, :3].astype(np.int32)) and pos.tobytes() == ref[:, 3:].copy().tobytes()


def test_cpp_two_view_triangulator_compiles(tmp_path):
    """the class layer and the data::keyframe adapter compile with g++ against the stand-in headers; without a GPU the program
    reports it (exit code 2) instead of failing"""
    import torch
    root = os.path.dirname(HERE)
    from openvslam_b200 import build
    build.build()
    libdir = os.path.join(root, "openvslam_b200", "lib")
    exe = str(tmp_path / "test_two_view_triangulator")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(HERE, "cpp", "standin"),
                           os.path.join(HERE, "cpp", "test_two_view_triangulator.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir,
                           "-o", exe])
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_two_view_triangulator_gpu.py")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
