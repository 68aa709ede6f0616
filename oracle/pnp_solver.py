"""ctypes front for the PnP RANSAC solver's oracle (oracle/pnp_solver_oracle.c, built into oracle/liboracle.so with the rest of
the oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports this module.
pose = {R row-major (9), t (3)} of cam_pose_cw: p_c = R p_w + t."""
import ctypes as C

import numpy as np

from .oracle import _p, lib

MIN_SET = 6


def ransac_sample(seed, k, n, m=MIN_SET):
    idx = (C.c_int * m)()
    lib().op_ransac_sample(C.c_uint64(int(seed) & (2 ** 64 - 1)), int(k), int(n), int(m), idx)
    return list(idx)


def jacobi(A):
    """-> (the final diagonal, V with the eigenvectors as columns)"""
    A = np.asarray(A, np.float64)
    N = A.shape[0]
    a, pa = _p(A.reshape(-1), np.float64)
    ev = np.zeros(N); V = np.zeros(N * N)
    lib().op_jacobi(N, pa, ev.ctypes.data_as(C.c_void_p), V.ctypes.data_as(C.c_void_p))
    return ev, V.reshape(N, N)


def max_cos(scale_factor):
    lib().op_max_cos.restype = C.c_double
    return float(lib().op_max_cos(C.c_float(scale_factor)))


def epnp(bearings, pos_w):
    b, pb = _p(np.asarray(bearings).reshape(-1, 3), np.float64); w, pw = _p(np.asarray(pos_w).reshape(-1, 3), np.float64)
    pose = np.zeros(12)
    lib().op_epnp(len(b), pb, pw, pose.ctypes.data_as(C.c_void_p))
    return pose


def pnp_solve_ransac(bearings, pos_w, scale_factor, min_num_inliers=10, max_num_iter=30, recompute=True, seed=0):
    """find_via_ransac on one problem -> dict(valid, pose_cw, num_inliers, best_iter, inliers[n], hyp_idx[max_num_iter, 6],
    hyp_pose[max_num_iter, 12], hyp_count[max_num_iter])"""
    b, pb = _p(np.asarray(bearings).reshape(-1, 3), np.float64); w, pw = _p(np.asarray(pos_w).reshape(-1, 3), np.float64)
    s, ps = _p(np.asarray(scale_factor).reshape(-1), np.float32)
    n = len(s)
    H = int(max_num_iter)
    pose = np.zeros(12); flags = np.zeros(max(n, 1), np.uint8)
    hidx = np.zeros(max(MIN_SET * H, 1), np.int32); hpose = np.zeros(max(12 * H, 1)); hcnt = np.zeros(max(H, 1), np.int32)
    valid, ninl, best = C.c_int(0), C.c_int(0), C.c_int(0)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib().op_pnp_solve_ransac(n, pb, pw, ps, int(min_num_inliers), H, int(bool(recompute)), C.c_uint64(int(seed) & (2 ** 64 - 1)),
                              vp(pose), C.byref(valid), C.byref(ninl), C.byref(best), vp(flags), vp(hidx), vp(hpose), vp(hcnt))
    return dict(valid=bool(valid.value), pose_cw=pose, num_inliers=ninl.value, best_iter=best.value, inliers=flags[:n].astype(bool),
                hyp_idx=hidx[:MIN_SET * H].reshape(H, MIN_SET), hyp_pose=hpose[:12 * H].reshape(H, 12), hyp_count=hcnt[:H].copy())
