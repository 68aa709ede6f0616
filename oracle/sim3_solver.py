"""ctypes front for the Sim3 RANSAC solver's oracle (oracle/sim3_solver_oracle.c, built into oracle/liboracle.so with the rest of
the oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports this module.
sim3 = {R row-major (9), t (3), s}, S p = s R p + t; S_12 maps keyframe 2's camera frame into keyframe 1's."""
import ctypes as C

import numpy as np

from .oracle import _p, camera, lib  # noqa: F401  (camera: built the same way as for the optimisers)


def splitmix64_mix(z):
    lib().os_splitmix64_mix.restype = C.c_uint64
    return int(lib().os_splitmix64_mix(C.c_uint64(int(z) & (2 ** 64 - 1))))


def ransac_triple(seed, k, n):
    idx = (C.c_int * 3)()
    lib().os_ransac_triple(C.c_uint64(int(seed) & (2 ** 64 - 1)), int(k), int(n), idx)
    return list(idx)


def jacobi4(A):
    """-> (eigenvalues[4] (the final diagonal), V[4, 4] with the eigenvectors as columns)"""
    A, pA = _p(np.asarray(A).reshape(16), np.float64)
    ev = np.zeros(4); V = np.zeros(16)
    lib().os_jacobi4(pA, ev.ctypes.data_as(C.c_void_p), V.ctypes.data_as(C.c_void_p))
    return ev, V.reshape(4, 4)


def horn(p1, p2, fix_scale=False):
    """p1, p2: (3, 3), one point per row -> (S12[13], S21[13])"""
    p1, pp1 = _p(np.asarray(p1).reshape(9), np.float64); p2, pp2 = _p(np.asarray(p2).reshape(9), np.float64)
    S12 = np.zeros(13); S21 = np.zeros(13)
    lib().os_horn(pp1, pp2, int(bool(fix_scale)), S12.ctypes.data_as(C.c_void_p), S21.ctypes.data_as(C.c_void_p))
    return S12, S21


def reproject(cam, rot, trans, p):
    """-> (ok, uv[2])"""
    rot, pr = _p(np.asarray(rot).reshape(9), np.float64); trans, pt = _p(trans, np.float64); p, pp = _p(p, np.float64)
    uv = np.zeros(2)
    ok = lib().os_reproject(C.byref(cam), pr, pt, pp, uv.ctypes.data_as(C.c_void_p))
    return bool(ok), uv


def sim3_solve_ransac(cam_1, cam_2, pose_1w, pose_2w, pos_w_1, sigma_sq_1, pos_w_2, sigma_sq_2, fix_scale, min_num_inliers=20,
                      max_num_iter=200, seed=0):
    """find_via_ransac on one problem -> dict(valid, sim3_12, num_inliers, best_iter, inliers[n], hyp_idx[max_num_iter, 3],
    hyp_count[max_num_iter])"""
    p1, pp1 = _p(np.asarray(pose_1w).reshape(12), np.float64); p2, pp2 = _p(np.asarray(pose_2w).reshape(12), np.float64)
    w1, pw1 = _p(np.asarray(pos_w_1).reshape(-1, 3), np.float64); s1, ps1 = _p(sigma_sq_1, np.float32)
    w2, pw2 = _p(np.asarray(pos_w_2).reshape(-1, 3), np.float64); s2, ps2 = _p(sigma_sq_2, np.float32)
    n = len(s1)
    H = int(max_num_iter)
    S = np.zeros(13); flags = np.zeros(max(n, 1), np.uint8)
    hidx = np.zeros(max(3 * H, 1), np.int32); hcnt = np.zeros(max(H, 1), np.int32)
    valid, ninl, best = C.c_int(0), C.c_int(0), C.c_int(0)
    lib().os_sim3_solve_ransac(C.byref(cam_1), C.byref(cam_2), pp1, pp2, n, pw1, ps1, pw2, ps2, int(bool(fix_scale)), int(min_num_inliers),
                               H, C.c_uint64(int(seed) & (2 ** 64 - 1)), S.ctypes.data_as(C.c_void_p), C.byref(valid), C.byref(ninl),
                               C.byref(best), flags.ctypes.data_as(C.c_void_p), hidx.ctypes.data_as(C.c_void_p),
                               hcnt.ctypes.data_as(C.c_void_p))
    return dict(valid=bool(valid.value), sim3_12=S, num_inliers=ninl.value, best_iter=best.value, inliers=flags[:n].astype(bool),
                hyp_idx=hidx[:3 * H].reshape(H, 3), hyp_count=hcnt[:H].copy())
