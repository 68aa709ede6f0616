"""ctypes front for the homography / fundamental-matrix RANSAC solvers' oracle (oracle/two_view_solver_oracle.c, built into
oracle/liboracle.so with the rest of the oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports
this module.  Keypoints are (n, 2) float32 pixel coordinates; matches_12 (m, 2) pairs (idx_1, idx_2) into them; H_21 maps view 1 to
view 2 (p2 ~ H_21 p1), F_21 satisfies p2^T F_21 p1 = 0."""
import ctypes as C

import numpy as np

from .oracle import _p, lib

MIN_SET = 8
MODELS = {"H": 0, "F": 1}


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def normalize(xy):
    """-> (normalised (n, 2) float32, (mean_x, mean_y, inv_x, inv_y) float32)"""
    xy, pxy = _p(np.asarray(xy).reshape(-1, 2), np.float32)
    out = np.zeros((max(len(xy), 1), 2), np.float32)
    T4 = np.zeros(4, np.float32)
    lib().ot_normalize(len(xy), pxy, _vp(out), _vp(T4))
    return out[:len(xy)], T4


def compute(model, norm_1, norm_2, matches_12, T4_1, T4_2, idx=None):
    """the model on the matches idx (None: all) from normalised points and both views' normalisation"""
    n1, pn1 = _p(np.asarray(norm_1).reshape(-1, 2), np.float32); n2, pn2 = _p(np.asarray(norm_2).reshape(-1, 2), np.float32)
    pr, ppr = _p(np.asarray(matches_12).reshape(-1, 2), np.int32)
    t1, pt1 = _p(T4_1, np.float32); t2, pt2 = _p(T4_2, np.float32)
    M = np.zeros(9)
    if idx is None:
        lib().ot_compute(MODELS[model], len(pr), pn1, pn2, ppr, None, pt1, pt2, _vp(M))
    else:
        ix, pix = _p(np.asarray(idx).reshape(-1), np.int32)
        lib().ot_compute(MODELS[model], len(ix), pn1, pn2, ppr, pix, pt1, pt2, _vp(M))
    return M.reshape(3, 3)


def check_inliers(model, M, keypts_1, keypts_2, matches_12, sigma=1.0):
    """-> (count, flags[m], score)"""
    M, pM = _p(np.asarray(M).reshape(9), np.float64)
    k1, pk1 = _p(np.asarray(keypts_1).reshape(-1, 2), np.float32); k2, pk2 = _p(np.asarray(keypts_2).reshape(-1, 2), np.float32)
    pr, ppr = _p(np.asarray(matches_12).reshape(-1, 2), np.int32)
    flags = np.zeros(max(len(pr), 1), np.uint8)
    score = C.c_double(0.0)
    cnt = lib().ot_check_inliers(MODELS[model], pM, len(pr), pk1, pk2, ppr, C.c_float(sigma), _vp(flags), C.byref(score))
    return cnt, flags[:len(pr)].astype(bool), score.value


def solve_ransac(model, keypts_1, keypts_2, matches_12, max_num_iter, recompute=True, seed=0, sigma=1.0):
    """find_via_ransac on one problem -> dict(valid, M (3, 3), num_inliers, best_iter, best_score, inliers[m],
    hyp_idx[max_num_iter, 8], hyp_M[max_num_iter, 3, 3], hyp_score[max_num_iter], hyp_count[max_num_iter])"""
    k1, pk1 = _p(np.asarray(keypts_1).reshape(-1, 2), np.float32); k2, pk2 = _p(np.asarray(keypts_2).reshape(-1, 2), np.float32)
    pr, ppr = _p(np.asarray(matches_12).reshape(-1, 2), np.int32)
    n = len(pr)
    H = int(max_num_iter)
    M = np.zeros(9); flags = np.zeros(max(n, 1), np.uint8)
    hidx = np.zeros(max(MIN_SET * H, 1), np.int32); hM = np.zeros(max(9 * H, 1)); hsc = np.zeros(max(H, 1)); hcnt = np.zeros(max(H, 1), np.int32)
    valid, ninl, best, score = C.c_int(0), C.c_int(0), C.c_int(0), C.c_double(0.0)
    lib().ot_solve_ransac(MODELS[model], len(k1), pk1, len(k2), pk2, n, ppr, C.c_float(sigma), H, int(bool(recompute)),
                          C.c_uint64(int(seed) & (2 ** 64 - 1)), _vp(M), C.byref(valid), C.byref(ninl), C.byref(best), C.byref(score),
                          _vp(flags), _vp(hidx), _vp(hM), _vp(hsc), _vp(hcnt))
    return dict(valid=bool(valid.value), M=M.reshape(3, 3), num_inliers=ninl.value, best_iter=best.value, best_score=score.value,
                inliers=flags[:n].astype(bool), hyp_idx=hidx[:MIN_SET * H].reshape(H, MIN_SET), hyp_M=hM[:9 * H].reshape(H, 3, 3),
                hyp_score=hsc[:H].copy(), hyp_count=hcnt[:H].copy())


def homography_solve_ransac(keypts_1, keypts_2, matches_12, max_num_iter, recompute=True, seed=0, sigma=1.0):
    r = solve_ransac("H", keypts_1, keypts_2, matches_12, max_num_iter, recompute, seed, sigma)
    r["H_21"] = r["M"]
    return r


def fundamental_solve_ransac(keypts_1, keypts_2, matches_12, max_num_iter, recompute=True, seed=0, sigma=1.0):
    r = solve_ransac("F", keypts_1, keypts_2, matches_12, max_num_iter, recompute, seed, sigma)
    r["F_21"] = r["M"]
    return r
