"""Host-side mirror of openvslam::module::two_view_triangulator (module/two_view_triangulator.h) and of the compute step of
mapping_module::create_new_landmarks (module/mapping_module.cc; names as recalled in SURVEY.md) over the C ABI of libovs_b200.so:
ovs_two_view_triangulate_host and ovs_create_new_landmarks_host."""
import ctypes as C

import numpy as np

from . import _lib
from .match import _matcher_handle
from .optimize import Camera

KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"), ("octave", "<i4"),
                           ("class_id", "<i4")])


class KeyframeView(C.Structure):
    _fields_ = [("pose_cw", C.c_double * 12), ("camera", Camera), ("true_baseline", C.c_double), ("scale_factor", C.c_float),
                ("num_scale_levels", C.c_int32), ("scale_factors", C.c_void_p), ("level_sigma_sq", C.c_void_p), ("num_keypts", C.c_int32),
                ("undist_keypts", C.c_void_p), ("bearings", C.c_void_p), ("stereo_x_right", C.c_void_p), ("depths", C.c_void_p),
                ("descriptors", C.c_void_p), ("has_landmark", C.c_void_p), ("bow_node", C.c_void_p)]


NEW_LANDMARK_DTYPE = np.dtype([("neighbour", "<i4"), ("idx_1", "<i4"), ("idx_2", "<i4"), ("reserved", "<i4"), ("pos_w", "<f8", (3,))])   # ovs_new_landmark


class keyframe:
    """What the triangulator and the triangulation matcher read of a data::keyframe.
    pose_cw: (3, 4) or 12 values {R row-major, t} of get_cam_pose(); camera: optimize.camera(...); scale_factor: scale_factor_;
    scale_factors / level_sigma_sq: the keyframe's tables; x, y, octave, angle: undist_keypts_; bearings: (n, 3) bearings_;
    stereo_x_right / depths: None for a monocular keyframe; true_baseline: camera_->true_baseline_;
    descriptors (n, 32), has_landmark (n), bow_node (n, < 0 = none): for create_new_landmarks."""

    def __init__(self, pose_cw, camera, scale_factor, scale_factors, level_sigma_sq, x, y, octave, bearings, angle=None,
                 stereo_x_right=None, depths=None, true_baseline=0.0, descriptors=None, has_landmark=None, bow_node=None):
        self.pose_cw = np.ascontiguousarray(pose_cw, np.float64).reshape(12)
        self.camera = camera
        self.scale_factor = float(scale_factor)
        self.scale_factors = np.ascontiguousarray(scale_factors, np.float32)
        self.level_sigma_sq = np.ascontiguousarray(level_sigma_sq, np.float32)
        n = len(np.asarray(x))
        kp = np.zeros(n, KEYPOINT_DTYPE)
        kp["x"] = x; kp["y"] = y; kp["octave"] = octave
        if angle is not None:
            kp["angle"] = angle
        self.keypts = kp
        self.bearings = np.ascontiguousarray(bearings, np.float64).reshape(n, 3)
        self.stereo_x_right = None if stereo_x_right is None else np.ascontiguousarray(stereo_x_right, np.float32)
        self.depths = None if depths is None else np.ascontiguousarray(depths, np.float32)
        self.true_baseline = float(true_baseline)
        self.descriptors = None if descriptors is None else np.ascontiguousarray(descriptors, np.uint8).reshape(n, 32)
        self.has_landmark = None if has_landmark is None else np.ascontiguousarray(has_landmark, np.uint8)
        self.bow_node = None if bow_node is None else np.ascontiguousarray(bow_node, np.int32)
        for a in (self.stereo_x_right, self.depths, self.has_landmark, self.bow_node):
            if a is not None and len(a) != n:
                raise ValueError("keyframe: one entry per keypoint")

    @property
    def num_keypts(self):
        return len(self.keypts)

    def view(self):
        """the ovs_keyframe_view of this keyframe (valid while the keyframe lives)"""
        def p(a):
            return None if a is None or a.size == 0 else a.ctypes.data
        v = KeyframeView()
        v.pose_cw[:] = self.pose_cw.tolist()
        v.camera = self.camera
        v.true_baseline = self.true_baseline
        v.scale_factor = self.scale_factor
        v.num_scale_levels = len(self.scale_factors)
        v.scale_factors = p(self.scale_factors); v.level_sigma_sq = p(self.level_sigma_sq)
        v.num_keypts = self.num_keypts
        v.undist_keypts = p(self.keypts); v.bearings = p(self.bearings)
        v.stereo_x_right = p(self.stereo_x_right); v.depths = p(self.depths)
        v.descriptors = p(self.descriptors); v.has_landmark = p(self.has_landmark); v.bow_node = p(self.bow_node)
        return v


def _views(kfs):
    arr = (KeyframeView * max(len(kfs), 1))()
    for i, k in enumerate(kfs):
        arr[i] = k.view()
    return arr


class two_view_triangulator(_matcher_handle):
    """module::two_view_triangulator(keyfrm_1, keyfrm_2, rays_parallax_deg_thr) batched over keyframe pairs: one device call
    triangulates every pair of every problem.  rays_parallax_deg_thr: create_new_landmarks passes 1.0."""

    def __init__(self, rays_parallax_deg_thr=1.0, device=0):
        super().__init__(device)
        self.rays_parallax_deg_thr_ = float(rays_parallax_deg_thr)

    def triangulate(self, problems):
        """problems: [(keyfrm_1, keyfrm_2, pairs (m, 2) of (idx_1, idx_2))] -> [(valid (m,) bool, pos_w (m, 3))] per problem;
        pos_w is zero where the pair makes no landmark."""
        B = len(problems)
        pairs = [np.ascontiguousarray(pr, np.int32).reshape(-1, 2) for _, _, pr in problems]
        off = np.zeros(B + 1, np.int32)
        off[1:] = np.cumsum([len(p) for p in pairs]) if B else []
        M = int(off[-1])
        allp = np.ascontiguousarray(np.concatenate(pairs) if M else np.zeros((1, 2), np.int32), np.int32)
        k1 = _views([p[0] for p in problems]); k2 = _views([p[1] for p in problems])
        valid = np.zeros(max(M, 1), np.uint8); pos = np.zeros((max(M, 1), 3))
        _lib.check(_lib.lib().ovs_two_view_triangulate_host(self._h, B, k1, k2, off.ctypes.data_as(C.c_void_p), allp.ctypes.data_as(C.c_void_p),
                                                            C.c_double(self.rays_parallax_deg_thr_), valid.ctypes.data_as(C.c_void_p),
                                                            pos.ctypes.data_as(C.c_void_p)))
        return [(valid[off[b]:off[b + 1]].astype(bool), pos[off[b]:off[b + 1]]) for b in range(B)]


def create_new_landmarks(matcher, keyfrm_1, neighbours, E_12, epipole_in_2, check_orientation=False, rays_parallax_deg_thr=1.0):
    """The compute step of mapping_module::create_new_landmarks on a matcher handle (match.robust or two_view_triangulator):
    for each neighbour in order, robust::match_for_triangulation with keyframe 1's landmark flags as they stand, then the
    triangulator on its pairs; a keypoint that gets a landmark is no query for the neighbours after it.
    E_12: (B, 3, 3); epipole_in_2: (B, 3).  -> records (r, 3) int32 (neighbour, idx_1, idx_2) and pos_w (r, 3), creation order."""
    B = len(neighbours)
    n1 = keyfrm_1.num_keypts
    E, pE = _f64(np.reshape(E_12, (-1,)) if B else np.zeros(9))
    ep, pep = _f64(np.reshape(epipole_in_2, (-1,)) if B else np.zeros(3))
    if B and (E.size != 9 * B or ep.size != 3 * B):
        raise ValueError("create_new_landmarks: one E_12 and one epipole per neighbour")
    k1 = _views([keyfrm_1]); k2 = _views(neighbours)
    out = np.zeros(max(n1, 1), NEW_LANDMARK_DTYPE)
    n = C.c_int(0)
    _lib.check(_lib.lib().ovs_create_new_landmarks_host(matcher._h, k1, B, k2, pE, pep, int(bool(check_orientation)),
                                                        C.c_double(rays_parallax_deg_thr), out.ctypes.data_as(C.c_void_p), n1, C.byref(n)))
    out = out[:n.value]
    rec = np.stack([out["neighbour"], out["idx_1"], out["idx_2"]], 1).astype(np.int32)
    return rec, out["pos_w"].copy()


def _f64(a):
    a = np.ascontiguousarray(a, np.float64)
    return a, a.ctypes.data_as(C.c_void_p)
