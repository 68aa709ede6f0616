"""ctypes front for the essential-matrix RANSAC solver's oracle (oracle/essential_solver_oracle.c, built into oracle/liboracle.so
with the rest of the oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports this module.
A match is a pair of unit bearings (b1 in camera 1, b2 in camera 2); E_21 (3 x 3) satisfies b2^T E_21 b1 = 0."""
import ctypes as C

import numpy as np

from .oracle import _p, lib, robust_brute_force_match

MIN_SET = 8


def compute_E(bearings_1, bearings_2, idx=None):
    b1, p1 = _p(np.asarray(bearings_1).reshape(-1, 3), np.float64); b2, p2 = _p(np.asarray(bearings_2).reshape(-1, 3), np.float64)
    E = np.zeros(9)
    if idx is None:
        lib().oe_compute_E(len(b1), p1, p2, None, E.ctypes.data_as(C.c_void_p))
    else:
        ix, pix = _p(np.asarray(idx).reshape(-1), np.int32)
        lib().oe_compute_E(len(ix), p1, p2, pix, E.ctypes.data_as(C.c_void_p))
    return E.reshape(3, 3)


def check_inliers(E, bearings_1, bearings_2):
    """-> (count, flags[n], score)"""
    E, pE = _p(np.asarray(E).reshape(9), np.float64)
    b1, p1 = _p(np.asarray(bearings_1).reshape(-1, 3), np.float64); b2, p2 = _p(np.asarray(bearings_2).reshape(-1, 3), np.float64)
    flags = np.zeros(max(len(b1), 1), np.uint8)
    score = C.c_double(0.0)
    cnt = lib().oe_check_inliers(pE, len(b1), p1, p2, flags.ctypes.data_as(C.c_void_p), C.byref(score))
    return cnt, flags[:len(b1)].astype(bool), score.value


def essential_solve_ransac(bearings_1, bearings_2, max_num_iter, recompute=True, seed=0):
    """find_via_ransac on one problem -> dict(valid, E_21 (3, 3), num_inliers, best_iter, best_score, inliers[n],
    hyp_idx[max_num_iter, 8], hyp_E[max_num_iter, 3, 3], hyp_score[max_num_iter], hyp_count[max_num_iter])"""
    b1, p1 = _p(np.asarray(bearings_1).reshape(-1, 3), np.float64); b2, p2 = _p(np.asarray(bearings_2).reshape(-1, 3), np.float64)
    n = len(b1)
    H = int(max_num_iter)
    E = np.zeros(9); flags = np.zeros(max(n, 1), np.uint8)
    hidx = np.zeros(max(MIN_SET * H, 1), np.int32); hE = np.zeros(max(9 * H, 1)); hsc = np.zeros(max(H, 1)); hcnt = np.zeros(max(H, 1), np.int32)
    valid, ninl, best, score = C.c_int(0), C.c_int(0), C.c_int(0), C.c_double(0.0)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib().oe_essential_solve_ransac(n, p1, p2, H, int(bool(recompute)), C.c_uint64(int(seed) & (2 ** 64 - 1)), vp(E), C.byref(valid),
                                    C.byref(ninl), C.byref(best), C.byref(score), vp(flags), vp(hidx), vp(hE), vp(hsc), vp(hcnt))
    return dict(valid=bool(valid.value), E_21=E.reshape(3, 3), num_inliers=ninl.value, best_iter=best.value, best_score=score.value,
                inliers=flags[:n].astype(bool), hyp_idx=hidx[:MIN_SET * H].reshape(H, MIN_SET), hyp_E=hE[:9 * H].reshape(H, 3, 3),
                hyp_score=hsc[:H].copy(), hyp_count=hcnt[:H].copy())


def robust_match_frame_and_keyframe(desc_frm, bearings_frm, desc_keyfrm, bearings_keyfrm, lm_valid_2=None, lowe_ratio=0.6,
                                    max_num_iter=50, seed=0):
    """match::robust::match_frame_and_keyframe: the oracle's brute force, then find_via_ransac(max_num_iter, false) on the pairs
    -> (num_inlier_matches, matched_keyfrm_idx_of_frm[n1])"""
    pairs = robust_brute_force_match(desc_frm, desc_keyfrm, lm_valid_2, lowe_ratio)
    n1 = len(np.asarray(desc_frm).reshape(-1, 32))
    out = np.full(n1, -1, np.int32)
    if len(pairs) < MIN_SET:
        return 0, out
    bf, bk = np.asarray(bearings_frm).reshape(-1, 3), np.asarray(bearings_keyfrm).reshape(-1, 3)
    r = essential_solve_ransac(bf[pairs[:, 0]], bk[pairs[:, 1]], max_num_iter, recompute=False, seed=seed)
    if not r["valid"]:
        return 0, out
    sel = pairs[r["inliers"]]
    out[sel[:, 0]] = sel[:, 1]
    return len(sel), out
