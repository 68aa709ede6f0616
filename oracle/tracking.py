"""ctypes front for the tracker's geometry oracle (oracle/tracking_oracle.c, built into oracle/liboracle.so with the rest of the
oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/; the product package never imports this module.  A geometry is
an openvslam_b200.match.FrameGeometry (the layout of ovs_frame_geometry)."""
import ctypes as C

import numpy as np

from .oracle import lib


def _p(a, dt):
    a = np.ascontiguousarray(a, dt)
    return a, a.ctypes.data_as(C.c_void_p)


def can_observe(geometry, pos_w, mean_normal, min_valid_dist, max_valid_dist, ray_cos_thr=0.5, usable=None):
    """frame::can_observe for every landmark, one after the other -> observable (n,) bool, reproj_xy (n, 2) f32, x_right (n,) f32,
    pred_scale_level (n,) i32 (zeros where not observable)."""
    pos, pp = _p(np.reshape(pos_w, (-1, 3)), np.float64)
    n = len(pos)
    nrm, pn = _p(np.reshape(mean_normal, (-1, 3)), np.float64)
    lo, plo = _p(min_valid_dist, np.float32); hi, phi = _p(max_valid_dist, np.float32)
    pu = None
    if usable is not None:
        usable, pu = _p(usable, np.uint8)
    ok = np.zeros(max(n, 1), np.uint8); uv = np.zeros((max(n, 1), 2), np.float32); xr = np.zeros(max(n, 1), np.float32)
    lv = np.zeros(max(n, 1), np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib().ott_can_observe_all(C.byref(geometry), n, pu, pp, pn, plo, phi, C.c_float(ray_cos_thr), vp(ok), vp(uv), vp(xr), vp(lv))
    return ok[:n].astype(bool), uv[:n], xr[:n], lv[:n]


def reproject(geometry, pos_w, usable=None):
    """camera::reproject_to_image for every landmark -> in_image (n,) bool, reproj_xy (n, 2) f32, x_right (n,) f32 (zeros where not
    in the image)."""
    pos, pp = _p(np.reshape(pos_w, (-1, 3)), np.float64)
    n = len(pos)
    pu = None
    if usable is not None:
        usable, pu = _p(usable, np.uint8)
    ok = np.zeros(max(n, 1), np.uint8); uv = np.zeros((max(n, 1), 2), np.float32); xr = np.zeros(max(n, 1), np.float32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib().ott_reproject_all(C.byref(geometry), n, pu, pp, vp(ok), vp(uv), vp(xr))
    return ok[:n].astype(bool), uv[:n], xr[:n]


def predict_scale_level(dist_f, max_valid_dist, log_scale_factor, num_levels):
    f = lib().ott_predict_scale_level
    f.argtypes = [C.c_float, C.c_float, C.c_float, C.c_int]
    return int(f(float(dist_f), float(max_valid_dist), float(log_scale_factor), int(num_levels)))


def motion_direction(pose_cw_curr, pose_cw_last, is_monocular, true_baseline):
    """-> (assume_forward, assume_backward)"""
    a, pa = _p(np.reshape(pose_cw_curr, 12), np.float64); b, pb = _p(np.reshape(pose_cw_last, 12), np.float64)
    fw = C.c_int(0); bw = C.c_int(0)
    lib().ott_motion_direction(pa, pb, int(bool(is_monocular)), C.c_double(true_baseline), C.byref(fw), C.byref(bw))
    return bool(fw.value), bool(bw.value)
