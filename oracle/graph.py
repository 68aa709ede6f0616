"""ctypes front for the pose-graph oracle (oracle/graph_oracle.c, built into oracle/liboracle.so with the rest of the oracle).
TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports this module.
sim3 = {R row-major (9), t (3), s}, S p = s R p + t; update = [omega (3), upsilon (3), sigma (1)], S <- exp(d) S."""
import ctypes as C

import numpy as np

from .oracle import BaStats, _p, _stats, lib


def _out(k):
    o = np.zeros(k)
    return o, o.ctypes.data_as(C.c_void_p)


def sim3_inverse(S):
    S, pS = _p(S, np.float64); o, po = _out(13)
    lib().ob_sim3_inverse(pS, po)
    return o


def sim3_compose(A, B):
    A, pA = _p(A, np.float64); B, pB = _p(B, np.float64); o, po = _out(13)
    lib().ob_sim3_compose(pA, pB, po)
    return o


def sim3_log(S):
    S, pS = _p(S, np.float64); o, po = _out(7)
    lib().ob_sim3_log(pS, po)
    return o


def sim3_adjoint(S):
    S, pS = _p(S, np.float64); o, po = _out(49)
    lib().ob_sim3_adjoint(pS, po)
    return o.reshape(7, 7)


def sim3_ad(xi):
    xi, px = _p(xi, np.float64); o, po = _out(49)
    lib().ob_sim3_ad(px, po)
    return o.reshape(7, 7)


def sim3_phi7(A):
    A, pA = _p(np.asarray(A).reshape(49), np.float64); o, po = _out(49)
    lib().ob_sim3_phi7(pA, po)
    return o.reshape(7, 7)


def graph_edge(S_ji, S_i, S_j):
    """-> (e[7], J[7, 14] = [J_i | J_j])"""
    a, pa = _p(S_ji, np.float64); b, pb = _p(S_i, np.float64); c, pc = _p(S_j, np.float64)
    e, pe = _out(7); J, pJ = _out(98)
    lib().ob_graph_edge(pa, pb, pc, pe, pJ)
    return e, J.reshape(7, 14)


def graph_optimize(sim3_cw, fixed, edge_i, edge_j, meas_ji, fix_scale, num_iter=50, lm_pos_w=None, lm_ref=None):
    """graph_optimizer::optimize -> (sim3_cw[K, 13], pose_cw[K, 12], lm_pos_w[L, 3], stats)"""
    S = np.array(sim3_cw, np.float64).reshape(-1, 13).copy()
    K = len(S)
    fixed, pf = _p(np.asarray(fixed).reshape(-1), np.uint8)
    ei, pi = _p(np.asarray(edge_i).reshape(-1), np.int32); ej, pj = _p(np.asarray(edge_j).reshape(-1), np.int32)
    meas, pm = _p(np.asarray(meas_ji, np.float64).reshape(-1, 13), np.float64)
    lm = np.zeros((0, 3)) if lm_pos_w is None else np.array(lm_pos_w, np.float64).reshape(-1, 3).copy()
    L = len(lm)
    ref, pr = _p(np.full(L, -1, np.int32) if lm_ref is None else np.asarray(lm_ref).reshape(-1), np.int32)
    pose = np.zeros((K, 12))
    st = BaStats()
    lib().ob_graph_optimize.restype = C.c_int
    rc = lib().ob_graph_optimize(K, S.ctypes.data_as(C.c_void_p), pf, len(ei), pi, pj, pm, int(bool(fix_scale)), int(num_iter), L,
                                 lm.ctypes.data_as(C.c_void_p), pr, pose.ctypes.data_as(C.c_void_p), C.byref(st))
    if rc != 0:
        raise ValueError("ob_graph_optimize: more free vertices than the dense solve takes")
    return S, pose, lm, _stats(st)
