"""ctypes front for the transform optimiser's oracle (oracle/sim3_oracle.c, built into oracle/liboracle.so with the rest of the
oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports this module.
sim3 = {R row-major (9), t (3), s}, S p = s R p + t; update = [omega (3), upsilon (3), sigma (1)]."""
import ctypes as C

import numpy as np

from .oracle import BaStats, _p, _stats, camera, lib  # noqa: F401  (camera: built the same way as for the other optimisers)


def sim3_exp(u):
    u, pu = _p(u, np.float64)
    out = np.zeros(13)
    lib().ob_sim3_exp(pu, out.ctypes.data_as(C.c_void_p))
    return out


def sim3_oplus(S, u, fix_scale=False):
    S, pS = _p(S, np.float64); u, pu = _p(u, np.float64)
    out = np.zeros(13)
    lib().ob_sim3_oplus(pS, pu, int(bool(fix_scale)), out.ctypes.data_as(C.c_void_p))
    return out


def sim3_edge(cam, S, pc, obs, forward=True):
    """forward: e = obs_1 - pi_1(S pc2); backward: e = obs_2 - pi_2(S^-1 pc1).  -> (e[2], J[2, 7])"""
    S, pS = _p(S, np.float64); pc, pp = _p(pc, np.float64); obs, po = _p(obs, np.float64)
    e = np.zeros(2); J = np.zeros(14)
    fn = lib().ob_sim3_edge_forward if forward else lib().ob_sim3_edge_backward
    fn(C.byref(cam), pS, pp, po, e.ctypes.data_as(C.c_void_p), J.ctypes.data_as(C.c_void_p))
    return e, J.reshape(2, 7)


def transform_optimize(cam_1, cam_2, pose_1w, pose_2w, pos_w_1, obs_xy_1, inv_sigma_sq_1, pos_w_2, obs_xy_2, inv_sigma_sq_2, sim3_12,
                       fix_scale, chi_sq=10.0, num_first_iter=5, num_iter=10):
    """transform_optimizer::optimize -> (num_inliers, sim3_12[13], inlier_flags[n], stats)"""
    p1, pp1 = _p(pose_1w, np.float64); p2, pp2 = _p(pose_2w, np.float64)
    w1, pw1 = _p(np.asarray(pos_w_1).reshape(-1, 3), np.float64); x1, px1 = _p(obs_xy_1, np.float32); s1, ps1 = _p(inv_sigma_sq_1, np.float32)
    w2, pw2 = _p(np.asarray(pos_w_2).reshape(-1, 3), np.float64); x2, px2 = _p(obs_xy_2, np.float32); s2, ps2 = _p(inv_sigma_sq_2, np.float32)
    n = len(s1)
    S = np.array(sim3_12, np.float64).reshape(13).copy()
    flags = np.zeros(max(n, 1), np.uint8)
    st = BaStats()
    lib().ob_transform_optimize.restype = C.c_int
    ninl = lib().ob_transform_optimize(C.byref(cam_1), C.byref(cam_2), pp1, pp2, n, pw1, px1, ps1, pw2, px2, ps2, int(bool(fix_scale)),
                                       C.c_float(chi_sq), int(num_first_iter), int(num_iter), S.ctypes.data_as(C.c_void_p),
                                       flags.ctypes.data_as(C.c_void_p), C.byref(st))
    return ninl, S, flags[:n].astype(bool), _stats(st)
