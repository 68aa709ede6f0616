"""ctypes front for the two-view triangulator's oracle (oracle/triangulation_oracle.c, built into oracle/liboracle.so with the rest
of the oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/; the product package never imports this module.  A keyframe is any
object with the attributes of openvslam_b200.module.keyframe (pose_cw, camera, true_baseline, scale_factor, scale_factors,
level_sigma_sq, keypts with x / y / angle / octave, bearings, stereo_x_right, depths, descriptors, has_landmark, bow_node)."""
import ctypes as C

import numpy as np

from .oracle import lib

REASONS = {0: "landmark", 1: "no branch", 2: "non-finite", 3: "cheirality 1", 4: "cheirality 2", 5: "reprojection 1", 6: "reprojection 2",
           7: "scale"}
BRANCHES = {-1: "none", 0: "two cameras", 1: "stereo 1", 2: "stereo 2"}


class _Camera(C.Structure):
    _fields_ = [("model", C.c_int), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("cols", C.c_double), ("rows", C.c_double)]


class _Keyframe(C.Structure):
    _fields_ = [("pose_cw", C.c_double * 12), ("camera", _Camera), ("true_baseline", C.c_double), ("scale_factor", C.c_float),
                ("num_scale_levels", C.c_int32), ("scale_factors", C.c_void_p), ("level_sigma_sq", C.c_void_p), ("num_keypts", C.c_int32),
                ("undist_keypts", C.c_void_p), ("bearings", C.c_void_p), ("stereo_x_right", C.c_void_p), ("depths", C.c_void_p),
                ("descriptors", C.c_void_p), ("has_landmark", C.c_void_p), ("bow_node", C.c_void_p)]


_KP = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])


def _kf(k, keep):
    def p(a, dt):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dt)
        keep.append(a)
        return a.ctypes.data if a.size else None
    kp = np.zeros(len(k.keypts), _KP)
    for f in ("x", "y", "angle", "octave"):
        kp[f] = k.keypts[f]
    v = _Keyframe()
    v.pose_cw[:] = [float(x) for x in np.reshape(k.pose_cw, 12)]
    c = k.camera
    v.camera = _Camera(c.model, c.fx, c.fy, c.cx, c.cy, c.focal_x_baseline, c.cols, c.rows)
    v.true_baseline = k.true_baseline; v.scale_factor = k.scale_factor
    v.num_scale_levels = len(k.scale_factors)
    v.scale_factors = p(k.scale_factors, np.float32); v.level_sigma_sq = p(k.level_sigma_sq, np.float32)
    v.num_keypts = len(kp)
    v.undist_keypts = p(kp, _KP); v.bearings = p(k.bearings, np.float64)
    v.stereo_x_right = p(k.stereo_x_right, np.float32); v.depths = p(k.depths, np.float32)
    v.descriptors = p(k.descriptors, np.uint8); v.has_landmark = p(k.has_landmark, np.uint8); v.bow_node = p(k.bow_node, np.int32)
    return v


def triangulate(keyfrm_1, keyfrm_2, pairs, rays_parallax_deg_thr=1.0):
    """-> valid (m,) bool, pos_w (m, 3) (zero where invalid), reason (m,) int (REASONS), branch (m,) int (BRANCHES)"""
    keep = []
    k1 = _kf(keyfrm_1, keep); k2 = _kf(keyfrm_2, keep)
    pr = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    m = len(pr)
    valid = np.zeros(max(m, 1), np.uint8); pos = np.zeros((max(m, 1), 3)); reason = np.zeros(max(m, 1), np.int32)
    branch = np.zeros(max(m, 1), np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib().otr_two_view_triangulate(C.byref(k1), C.byref(k2), m, vp(pr), C.c_double(rays_parallax_deg_thr), vp(valid), vp(pos), vp(reason),
                                   vp(branch))
    return valid[:m].astype(bool), pos[:m], reason[:m], branch[:m]


def create_new_landmarks(keyfrm_1, neighbours, E_12, epipole_in_2, check_orientation=False, rays_parallax_deg_thr=1.0):
    """the sequential loop over the neighbours -> records (r, 3) int32 (neighbour, idx_1, idx_2), pos_w (r, 3)"""
    keep = []
    k1 = _kf(keyfrm_1, keep)
    B = len(neighbours)
    k2 = (_Keyframe * max(B, 1))()
    for b, n in enumerate(neighbours):
        k2[b] = _kf(n, keep)
    E = np.ascontiguousarray(np.reshape(E_12, -1) if B else np.zeros(9), np.float64)
    ep = np.ascontiguousarray(np.reshape(epipole_in_2, -1) if B else np.zeros(3), np.float64)
    n1 = len(keyfrm_1.keypts)
    rec = np.zeros((max(n1, 1), 3), np.int32); pos = np.zeros((max(n1, 1), 3))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    r = lib().otr_create_new_landmarks(C.byref(k1), B, k2, vp(E), vp(ep), int(bool(check_orientation)), C.c_double(rays_parallax_deg_thr),
                                       vp(rec), vp(pos))
    return rec[:r], pos[:r]
