"""ctypes front for the fuse oracle (oracle/fuse_oracle.c, built into oracle/liboracle.so with the rest of the oracle).  TEST
INFRASTRUCTURE ONLY: imported by tests/ and tools/; the product package never imports this module.  A geometry is an
openvslam_b200.match.FrameGeometry (the layout of ott_geometry); a frame is an oracle.oracle.MatchFrame."""
import ctypes as C

import numpy as np

from .oracle import lib


def _p(a, dt):
    a = np.ascontiguousarray(a, dt)
    return a, a.ctypes.data_as(C.c_void_p)


def fuse_observe(geometry, pos_w, mean_normal, min_valid_dist, max_valid_dist):
    """The geometry of replace_duplication for every landmark -> passed (n,) bool, reproj_xy (n, 2) f64 (the unrounded
    reprojection), x_right (n,) f32, pred_level (n,) i32 (zeros where not passed)."""
    pos = np.ascontiguousarray(np.reshape(pos_w, (-1, 3)), np.float64)
    nrm = np.ascontiguousarray(np.reshape(mean_normal, (-1, 3)), np.float64)
    lo = np.ascontiguousarray(min_valid_dist, np.float32); hi = np.ascontiguousarray(max_valid_dist, np.float32)
    n = len(pos)
    f = lib().ott_fuse_observe
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    ok = np.zeros(n, bool); uv = np.zeros((n, 2), np.float64); xr = np.zeros(n, np.float32); lv = np.zeros(n, np.int32)
    for l in range(n):
        u = (C.c_double * 2)(); x = C.c_float(0.0); v = C.c_int(0)
        r = f(C.addressof(geometry), pos[l].ctypes.data, nrm[l].ctypes.data, float(lo[l]), float(hi[l]), C.addressof(u), C.addressof(x),
              C.addressof(v))
        if r:
            ok[l] = True; uv[l] = (u[0], u[1]); xr[l] = x.value; lv[l] = v.value
    return ok, uv, xr, lv


def replace_duplication(geometry, frame, scale_factors, inv_level_sigma_sq, q_lm, pos_w, mean_normal, min_valid_dist, max_valid_dist, lm_desc,
                        margin=3.0):
    """One target keyframe (geometry + oracle.oracle.MatchFrame of its keypoints) and its queries q_lm (landmark row or -1) ->
    (num_fused, best_idx (nq,), passed (nq,) bool, reproj_xy (nq, 2) f32, x_right (nq,) f32, pred_level (nq,) i32)."""
    ql, pql = _p(q_lm, np.int32)
    nq = len(ql)
    pos, pp = _p(np.reshape(pos_w, (-1, 3)), np.float64); nrm, pn = _p(np.reshape(mean_normal, (-1, 3)), np.float64)
    lo, plo = _p(min_valid_dist, np.float32); hi, phi = _p(max_valid_dist, np.float32)
    d, pd = _p(np.reshape(lm_desc, (-1, 32)), np.uint8)
    sf, psf = _p(scale_factors, np.float32); iw, piw = _p(inv_level_sigma_sq, np.float32)
    n1 = max(nq, 1)
    best = np.full(n1, -1, np.int32); ok = np.zeros(n1, np.uint8); uv = np.zeros((n1, 2), np.float32); xr = np.zeros(n1, np.float32)
    lv = np.zeros(n1, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    f = lib().ott_fuse_replace_duplication_all
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_float] + [C.c_void_p] * 5
    num = f(C.addressof(geometry), C.addressof(frame.c), psf, piw, nq, pql, pp, pn, plo, phi, pd, float(margin), vp(best), vp(ok), vp(uv),
            vp(xr), vp(lv))
    return num, best[:nq], ok[:nq].astype(bool), uv[:nq], xr[:nq], lv[:nq]
