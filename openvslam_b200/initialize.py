"""Host-side mirror of openvslam::initialize::perspective and initialize::bearing_vector (src/openvslam/initialize/*.h) over the C
ABI of libovs_b200.so: monocular map initialisation, from the area matches to the initial pose and triangulated points, solved on
the GPU for a whole batch of problems in one call (include/ovs_b200.h, ovs_initialize_*_host, for the field-by-field mapping).

A view is what the initialiser reads of a frame: `view(camera, keypts, bearings)` with an optimize.Camera, the undistorted keypoints
(n, 2) and their unit bearings (n, 3)."""
import ctypes as C
import types

import numpy as np

from . import _lib
from .match import _matcher_handle
from .optimize import Camera

STATUS = {0: "ok", 1: "no valid model", 2: "decomposition refused", 3: "too few", 4: "ambiguous", 5: "small parallax"}
MODEL = {0: None, 1: "H", 2: "F", 3: "E"}

# cv::KeyPoint / ovs_keypoint (28 bytes): the initialisers read pt only
_KEYPOINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"), ("octave", "<i4"),
                      ("class_id", "<i4")])


class InitView(C.Structure):
    _fields_ = [("camera", Camera), ("num_keypts", C.c_int32), ("undist_keypts", C.c_void_p), ("bearings", C.c_void_p)]


class InitResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("model", C.c_int32), ("chosen", C.c_int32), ("num_hypotheses", C.c_int32),
                ("num_valid", C.c_int32 * 8), ("cos_parallax", C.c_float * 8), ("rot_ref_to_cur", C.c_double * 9),
                ("trans_ref_to_cur", C.c_double * 3), ("solver_M", (C.c_double * 9) * 2), ("solver_score", C.c_double * 2),
                ("solver_num_inliers", C.c_int32 * 2), ("solver_valid", C.c_uint8 * 2), ("reserved", C.c_uint8 * 6)]


def view(camera, keypts, bearings):
    keypts = np.ascontiguousarray(np.asarray(keypts, np.float32).reshape(-1, 2))
    bearings = np.ascontiguousarray(np.asarray(bearings, np.float64).reshape(-1, 3))
    if len(keypts) != len(bearings):
        raise ValueError("view: one bearing per keypoint")
    return types.SimpleNamespace(camera=camera, keypts=keypts, bearings=bearings)


def _result(r, flags, pts):
    """one problem's outcome as a dict"""
    return dict(ok=r.status == 0, status=STATUS[r.status], status_code=r.status, model=MODEL[r.model], chosen=r.chosen,
                num_hypotheses=r.num_hypotheses, num_valid=np.array(r.num_valid[:], np.int32),
                cos_parallax=np.array(r.cos_parallax[:], np.float32),
                parallax_deg=np.degrees(np.arccos(np.clip(np.array(r.cos_parallax[:], np.float64), -1.0, 1.0))),
                rot_ref_to_cur=np.array(r.rot_ref_to_cur[:]).reshape(3, 3), trans_ref_to_cur=np.array(r.trans_ref_to_cur[:]),
                solver_M=np.array([r.solver_M[s][:] for s in range(2)]).reshape(2, 3, 3), solver_score=np.array(r.solver_score[:]),
                solver_num_inliers=np.array(r.solver_num_inliers[:], np.int32), solver_valid=np.array(r.solver_valid[:], bool),
                is_triangulated=flags.astype(bool), triangulated_pts=pts)


class _initializer(_matcher_handle):
    _entry = None

    def __init__(self, ref_view, num_ransac_iters=100, min_num_triangulated=50, parallax_deg_thr=1.0, reproj_err_thr_sq=4.0, device=0):
        super().__init__(device)
        self.ref_view_ = ref_view
        self.num_ransac_iters_ = int(num_ransac_iters)
        self.min_num_triangulated_ = int(min_num_triangulated)
        self.parallax_deg_thr_ = float(parallax_deg_thr)
        self.reproj_err_thr_sq_ = float(reproj_err_thr_sq)
        self.result_ = None

    def initialize_batch(self, problems, seeds=None):
        """problems: list of dicts with ref (a view), cur (a view) and ref_matches_with_cur (one entry per reference keypoint: the
        matched current keypoint or -1); seeds: one sampler seed per problem (default: the problem's index).  The constructor's
        settings apply to every problem.  Returns one dict per problem (ok, status, model, chosen, num_valid, cos_parallax,
        parallax_deg, rot_ref_to_cur, trans_ref_to_cur, solver_M / solver_score / solver_num_inliers / solver_valid,
        is_triangulated, triangulated_pts)."""
        B = len(problems)
        seeds = np.arange(B, dtype=np.uint64) if seeds is None else np.ascontiguousarray(seeds, np.uint64).reshape(-1)
        if len(seeds) != B:
            raise ValueError("one seed per problem")
        keep = []

        def flat(v):
            kp = np.zeros(max(len(v.keypts), 1), _KEYPOINT)
            kp["x"][:len(v.keypts)] = v.keypts[:, 0]; kp["y"][:len(v.keypts)] = v.keypts[:, 1]
            b = np.ascontiguousarray(v.bearings, np.float64)
            keep.extend((kp, b))
            return InitView(v.camera, len(v.keypts), kp.ctypes.data, b.ctypes.data if b.size else None)
        refs = (InitView * max(B, 1))(*[flat(p["ref"]) for p in problems])
        curs = (InitView * max(B, 1))(*[flat(p["cur"]) for p in problems])
        rm = [np.asarray(p["ref_matches_with_cur"], np.int32).reshape(-1) for p in problems]
        for p, r in zip(problems, rm):
            if len(r) != len(p["ref"].keypts):
                raise ValueError("ref_matches_with_cur needs one entry per reference keypoint")
        off = np.concatenate([[0], np.cumsum([len(r) for r in rm])]).astype(np.int64)
        K1 = int(off[-1])
        rmc = np.ascontiguousarray(np.concatenate(rm) if K1 else np.zeros(1, np.int32), np.int32)
        res = (InitResult * max(B, 1))()
        flags = np.zeros(max(K1, 1), np.uint8); pts = np.zeros((max(K1, 1), 3))
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(getattr(_lib.lib(), self._entry)(self._h, B, refs, curs, vp(rmc), self.num_ransac_iters_, self.min_num_triangulated_,
                                                    C.c_float(self.parallax_deg_thr_), C.c_float(self.reproj_err_thr_sq_),
                                                    vp(seeds if B else np.zeros(1, np.uint64)), res, vp(flags), vp(pts)))
        return [_result(res[b], flags[off[b]:off[b + 1]].copy(), pts[off[b]:off[b + 1]].copy()) for b in range(B)]

    def initialize(self, cur_view, ref_matches_with_cur, seed=0):
        """initialize(cur_frm, ref_matches_with_cur) on the constructor's reference view -> bool"""
        self.result_ = self.initialize_batch([dict(ref=self.ref_view_, cur=cur_view, ref_matches_with_cur=ref_matches_with_cur)], [seed])[0]
        return self.result_["ok"]

    def get_rotation_ref_to_cur(self):
        return self.result_["rot_ref_to_cur"]

    def get_translation_ref_to_cur(self):
        return self.result_["trans_ref_to_cur"]

    def get_triangulated_pts(self):
        return self.result_["triangulated_pts"]

    def get_triangulated_flags(self):
        return self.result_["is_triangulated"]


class perspective(_initializer):
    """openvslam::initialize::perspective(ref_frm, num_ransac_iters = 100, min_num_triangulated = 50, parallax_deg_thr = 1.0,
    reproj_err_thr = 4.0) for perspective (and fisheye, on undistorted keypoints) cameras: the homography and fundamental-matrix
    solvers, the model choice, the decomposition and check_pose on the GPU.  reproj_err_thr_sq is check_pose's squared pixel
    threshold (4.0 = 4 sigma^2 with sigma = 1)."""
    _entry = "ovs_initialize_perspective_host"


class bearing_vector(_initializer):
    """openvslam::initialize::bearing_vector(...) for equirectangular cameras: the essential solver on the bearings, 4 hypotheses and
    no depth test; the same interface as perspective."""
    _entry = "ovs_initialize_bearing_vector_host"
