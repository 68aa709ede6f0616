"""ctypes front for the map initialisers' oracle (oracle/initializer_oracle.c, built into oracle/liboracle.so with the rest of the
oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports this module.  A camera is a dict or object
with model (0 perspective, 1 equirectangular), fx, fy, cx, cy, cols, rows; keypoints are (n, 2) float32, bearings (n, 3) float64."""
import ctypes as C

import numpy as np

from .oracle import lib

REASONS = {-1: "unused hypothesis", 0: "valid", 1: "valid, small parallax", 2: "non-finite", 3: "depth (reference)", 4: "depth (current)",
           5: "reprojection (reference)", 6: "reprojection (current)", 7: "not a solver inlier"}


class _Camera(C.Structure):
    _fields_ = [("model", C.c_int), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("cols", C.c_double), ("rows", C.c_double)]


class Result(C.Structure):
    _fields_ = [("status", C.c_int32), ("model", C.c_int32), ("chosen", C.c_int32), ("num_hypotheses", C.c_int32),
                ("num_valid", C.c_int32 * 8), ("cos_parallax", C.c_float * 8), ("rot_ref_to_cur", C.c_double * 9),
                ("trans_ref_to_cur", C.c_double * 3), ("solver_M", (C.c_double * 9) * 2), ("solver_score", C.c_double * 2),
                ("solver_num_inliers", C.c_int32 * 2), ("solver_valid", C.c_uint8 * 2), ("reserved", C.c_uint8 * 6)]


def camera(c):
    g = (lambda k: c[k]) if isinstance(c, dict) else (lambda k: getattr(c, k))
    return _Camera(int(g("model")), float(g("fx")), float(g("fy")), float(g("cx")), float(g("cy")), 0.0, float(g("cols")), float(g("rows")))


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def svd3(A, third_by_cross=False):
    """-> U, d, V with A = U diag(d) V^T"""
    A = np.ascontiguousarray(A, np.float64).reshape(9)
    U = np.zeros(9); d = np.zeros(3); V = np.zeros(9)
    lib().oi_svd3(_vp(A), int(bool(third_by_cross)), _vp(U), _vp(d), _vp(V))
    return U.reshape(3, 3), d, V.reshape(3, 3)


def decompose_homography(H, cam_1, cam_2):
    """-> None when refused, else (R (8, 3, 3), t (8, 3), n (8, 3))"""
    H = np.ascontiguousarray(H, np.float64).reshape(9)
    R = np.zeros(72); t = np.zeros(24); n = np.zeros(24)
    c1, c2 = camera(cam_1), camera(cam_2)
    if not lib().oi_decompose_homography(_vp(H), C.byref(c1), C.byref(c2), _vp(R), _vp(t), _vp(n)):
        return None
    return R.reshape(8, 3, 3), t.reshape(8, 3), n.reshape(8, 3)


def decompose_essential(E):
    E = np.ascontiguousarray(E, np.float64).reshape(9)
    R = np.zeros(36); t = np.zeros(12)
    lib().oi_decompose_essential(_vp(E), _vp(R), _vp(t))
    return R.reshape(4, 3, 3), t.reshape(4, 3)


def decompose_fundamental(F, cam_1, cam_2):
    F = np.ascontiguousarray(F, np.float64).reshape(9)
    R = np.zeros(36); t = np.zeros(12)
    c1, c2 = camera(cam_1), camera(cam_2)
    lib().oi_decompose_fundamental(_vp(F), C.byref(c1), C.byref(c2), _vp(R), _vp(t))
    return R.reshape(4, 3, 3), t.reshape(4, 3)


def check_match(R, t, cam_ref, cam_cur, b_ref, b_cur, kp_ref, kp_cur, reproj_err_thr_sq=4.0, depth_is_positive=True):
    """-> (code (REASONS), p (3,), cos_parallax (float32))"""
    Rt = np.ascontiguousarray(np.concatenate([np.reshape(R, 9), np.reshape(t, 3)]), np.float64)
    b1 = np.ascontiguousarray(b_ref, np.float64); b2 = np.ascontiguousarray(b_cur, np.float64)
    k1 = np.ascontiguousarray(kp_ref, np.float32); k2 = np.ascontiguousarray(kp_cur, np.float32)
    p = np.zeros(3); cp = C.c_float(0.0)
    c1, c2 = camera(cam_ref), camera(cam_cur)
    code = lib().oi_check_match(_vp(Rt), C.byref(c1), C.byref(c2), _vp(b1), _vp(b2), _vp(k1), _vp(k2), C.c_double(reproj_err_thr_sq),
                                int(bool(depth_is_positive)), _vp(p), C.byref(cp))
    return code, p, np.float32(cp.value)


def initialize(perspective, cam_ref, cam_cur, keypts_ref, bearings_ref, keypts_cur, bearings_cur, ref_matches_with_cur,
               num_ransac_iters=100, min_num_triangulated=50, parallax_deg_thr=1.0, reproj_err_thr_sq=4.0, seed=0):
    """initialize() on one problem -> dict(result (Result), hyp_R (8, 3, 3), hyp_t (8, 3), reason (8, m) per hypothesis and match
    in reference-index order, is_triangulated (n_ref,) bool, triangulated_pts (n_ref, 3))"""
    k1 = np.ascontiguousarray(np.reshape(keypts_ref, (-1, 2)), np.float32); k2 = np.ascontiguousarray(np.reshape(keypts_cur, (-1, 2)), np.float32)
    b1 = np.ascontiguousarray(np.reshape(bearings_ref, (-1, 3)), np.float64); b2 = np.ascontiguousarray(np.reshape(bearings_cur, (-1, 3)), np.float64)
    rm = np.ascontiguousarray(ref_matches_with_cur, np.int32).reshape(-1)
    n1, m = len(k1), int((rm >= 0).sum())
    res = Result()
    hR = np.zeros(72); ht = np.zeros(24); reason = np.zeros(max(8 * m, 1), np.int32)
    flags = np.zeros(max(n1, 1), np.uint8); pts = np.zeros((max(n1, 1), 3))
    c1, c2 = camera(cam_ref), camera(cam_cur)
    lib().oi_initialize(int(bool(perspective)), C.byref(c1), C.byref(c2), n1, _vp(k1), _vp(b1), len(k2), _vp(k2), _vp(b2), _vp(rm),
                        int(num_ransac_iters), int(min_num_triangulated), C.c_float(parallax_deg_thr), C.c_float(reproj_err_thr_sq),
                        C.c_uint64(int(seed) & (2 ** 64 - 1)), C.byref(res), _vp(hR), _vp(ht), _vp(reason), _vp(flags), _vp(pts))
    return dict(result=res, hyp_R=hR.reshape(8, 3, 3), hyp_t=ht.reshape(8, 3), reason=reason[:8 * m].reshape(8, m),
                is_triangulated=flags[:n1].astype(bool), triangulated_pts=pts[:n1])
