"""Host-side mirror of openvslam::match::* (src/openvslam/match/{base,robust,...}.h; names as
recalled in SURVEY.md 8a) over the C ABI of libovs_b200.so."""
import ctypes as C
import numpy as np

from . import _lib
from .optimize import Camera

HAMMING_DIST_THR_LOW = 50
HAMMING_DIST_THR_HIGH = 100
MAX_HAMMING_DIST = 256


class _matcher_handle:
    def __init__(self, device=0):
        self._h = C.c_void_p()
        self._indexes = set()      # handles of the frame indexes built on this matcher and not yet destroyed
        _lib.check(_lib.lib().ovs_matcher_create(int(device), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            # an index uses its matcher until it is destroyed, and the garbage collector may finalize a matcher before
            # the indexes that refer to it: destroy those first
            for h in getattr(self, "_indexes", ()):
                _lib.lib().ovs_frame_index_destroy(C.c_void_p(h))
            self._indexes = set()
            _lib.lib().ovs_matcher_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def num_requeries(self):
        v = C.c_int(0)
        _lib.check(_lib.lib().ovs_matcher_num_requeries(self._h, C.byref(v)))
        return v.value

    def last_kernel_us(self):
        v = C.c_float(0)
        _lib.check(_lib.lib().ovs_matcher_last_kernel_us(self._h, C.byref(v)))
        return v.value


def _desc(a):
    a = np.ascontiguousarray(a, np.uint8).reshape(-1, 32)
    return a, a.ctypes.data_as(C.c_void_p)


class robust(_matcher_handle):
    """openvslam::match::robust (lowe_ratio_, check_orientation_)."""

    def __init__(self, lowe_ratio=0.6, check_orientation=True, device=0):
        super().__init__(device)
        self.lowe_ratio_ = float(lowe_ratio)
        self.check_orientation_ = bool(check_orientation)

    def brute_force_topk(self, query, train):
        q, pq = _desc(query); t, pt = _desc(train)
        keys = np.zeros((len(q), 8), np.uint32)
        _lib.check(_lib.lib().ovs_match_bruteforce_topk_host(self._h, pq, len(q), pt, len(t), keys.ctypes.data_as(C.c_void_p)))
        return keys

    def brute_force_nearest(self, desc1, desc2):
        d1, p1 = _desc(desc1); d2, p2 = _desc(desc2)
        bi = np.zeros(len(d1), np.int32); bd = np.zeros(len(d1), np.int32); sd = np.zeros(len(d1), np.int32)
        _lib.check(_lib.lib().ovs_match_bruteforce_host(self._h, p1, len(d1), p2, len(d2), bi.ctypes.data_as(C.c_void_p),
                                                        bd.ctypes.data_as(C.c_void_p), sd.ctypes.data_as(C.c_void_p)))
        return bi, bd, sd

    def brute_force_match(self, desc_frm, desc_keyfrm, lm_valid_2=None):
        """robust::brute_force_match(frm, keyfrm, matches) -> matches[(idx_1, idx_2)]."""
        d1, p1 = _desc(desc_frm); d2, p2 = _desc(desc_keyfrm)
        vp = None
        if lm_valid_2 is not None:
            lm_valid_2 = np.ascontiguousarray(lm_valid_2, np.uint8)
            vp = lm_valid_2.ctypes.data_as(C.c_void_p)
        cap = max(min(len(d1), len(d2)), 1)
        pairs = np.zeros((cap, 2), np.int32)
        n = C.c_int(0)
        _lib.check(_lib.lib().ovs_robust_brute_force_match_host(self._h, p1, len(d1), p2, len(d2), vp, C.c_float(self.lowe_ratio_),
                                                                pairs.ctypes.data_as(C.c_void_p), cap, C.byref(n)))
        return pairs[:n.value].copy()

    def brute_force_match_device(self, d_desc_frm, n1, d_desc_keyfrm, n2, lm_valid_2=None):
        """The same on descriptors resident in device memory (device pointers as ints, 16-byte aligned)."""
        vp = None
        if lm_valid_2 is not None:
            lm_valid_2 = np.ascontiguousarray(lm_valid_2, np.uint8)
            vp = lm_valid_2.ctypes.data_as(C.c_void_p)
        cap = max(min(int(n1), int(n2)), 1)
        pairs = np.zeros((cap, 2), np.int32)
        n = C.c_int(0)
        _lib.check(_lib.lib().ovs_robust_brute_force_match_device(self._h, C.c_void_p(int(d_desc_frm)), int(n1), C.c_void_p(int(d_desc_keyfrm)), int(n2), vp,
                                                                  C.c_float(self.lowe_ratio_), pairs.ctypes.data_as(C.c_void_p), cap, C.byref(n)))
        return pairs[:n.value].copy()

    def brute_force_topk_device(self, d_query, nq, d_train, nt, d_keys_out):
        """ovs_match_bruteforce_topk_device: brute_force_topk's (nq, 8) uint32 keys written to d_keys_out, with the descriptors
        in device memory (device pointers as ints, descriptors 16-byte aligned); returns when the keys are written."""
        _lib.check(_lib.lib().ovs_match_bruteforce_topk_device(self._h, C.c_void_p(int(d_query)), int(nq), C.c_void_p(int(d_train)), int(nt),
                                                               C.c_void_p(int(d_keys_out))))

    def match_frame_and_keyframe(self, desc_frm, bearings_frm, desc_keyfrm, bearings_keyfrm, lm_valid_2=None, max_num_iter=50, seed=0):
        """robust::match_frame_and_keyframe(frm, keyfrm, matched_lms_in_frm): brute_force_match, then the essential-matrix RANSAC on
        the pairs (find_via_ransac(max_num_iter, false)) -> (num_inlier_matches, matched_keyfrm_idx_of_frm[n1]): the keyframe keypoint
        whose landmark frame keypoint i receives, or -1.  bearings_*: (n, 3) unit bearings (frm.bearings_, keyfrm->bearings_)."""
        d1, p1 = _desc(desc_frm); d2, p2 = _desc(desc_keyfrm)
        b1, pb1 = _f64(bearings_frm); b2, pb2 = _f64(bearings_keyfrm)
        if b1.size != 3 * len(d1) or b2.size != 3 * len(d2):
            raise ValueError("match_frame_and_keyframe: one bearing (3 doubles) per keypoint")
        _keep, vp = _u8p(lm_valid_2)
        out = np.full(max(len(d1), 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_robust_match_frame_and_keyframe_host(self._h, p1, pb1, len(d1), p2, pb2, len(d2), vp, C.c_float(self.lowe_ratio_),
                                                                       int(max_num_iter), C.c_uint64(int(seed) & (2 ** 64 - 1)),
                                                                       out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:len(d1)]

    def match_frame_and_keyframe_device(self, d_desc_frm, d_bearings_frm, n1, d_desc_keyfrm, d_bearings_keyfrm, n2, lm_valid_2=None,
                                        max_num_iter=50, seed=0):
        """The same on descriptors and bearings resident in device memory (device pointers as ints; the outputs of extract_device
        and undistort_keypoints_device): only the pair list goes to the device and the flags come back."""
        _keep, vp = _u8p(lm_valid_2)
        out = np.full(max(int(n1), 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_robust_match_frame_and_keyframe_device(self._h, C.c_void_p(int(d_desc_frm)), C.c_void_p(int(d_bearings_frm)), int(n1),
                                                                         C.c_void_p(int(d_desc_keyfrm)), C.c_void_p(int(d_bearings_keyfrm)), int(n2), vp,
                                                                         C.c_float(self.lowe_ratio_), int(max_num_iter),
                                                                         C.c_uint64(int(seed) & (2 ** 64 - 1)), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:int(n1)]

    def match_for_triangulation(self, desc_1, bearing_1, octave_1, angle_1, has_lm_1, is_stereo_1, bow_node_1,
                                desc_2, bearing_2, angle_2, has_lm_2, is_stereo_2, bow_node_2, E_12, epipole_in_2, scale_factors_1):
        """robust::match_for_triangulation(keyfrm_1, keyfrm_2, E_12, matched_idx_pairs) -> (num_matches, matched_idx_2_of_1[n1]);
        the BoW feature vectors come in as per-keypoint node ids."""
        d1, pd1 = _desc(desc_1); b1, pb1 = _f64(bearing_1); o1, po1 = _i32(octave_1); a1, pa1 = _f32(angle_1)
        _keep1, pl1 = _u8p(has_lm_1); _keep2, ps1 = _u8p(is_stereo_1); n1, pn1 = _i32(bow_node_1)
        d2, pd2 = _desc(desc_2); b2, pb2 = _f64(bearing_2); a2, pa2 = _f32(angle_2)
        _keep3, pl2 = _u8p(has_lm_2); _keep4, ps2 = _u8p(is_stereo_2); n2, pn2 = _i32(bow_node_2)
        E, pE = _f64(E_12); ep, pep = _f64(epipole_in_2); sf, psf = _f32(scale_factors_1)
        out = np.full(max(len(o1), 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_robust_match_for_triangulation_host(self._h, len(o1), pd1, pb1, po1, pa1, pl1, ps1, pn1, len(a2), pd2, pb2, pa2, pl2, ps2,
                                                                      pn2, pE, pep, psf, len(sf), int(self.check_orientation_),
                                                                      out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:len(o1)]


# ------------------------------------------------------------------ windowed matchers
class Grid(C.Structure):
    _fields_ = [("min_x", C.c_float), ("min_y", C.c_float), ("inv_cell_width", C.c_float), ("inv_cell_height", C.c_float),
                ("num_grid_cols", C.c_int32), ("num_grid_rows", C.c_int32)]


def camera_grid(min_x, max_x, min_y, max_y, num_grid_cols=64, num_grid_rows=48):
    """camera::base: inv_cell_width_ = num_grid_cols_ / (img_bounds_.max_x_ - img_bounds_.min_x_) (float)."""
    return Grid(min_x, min_y, np.float32(float(num_grid_cols) / (max_x - min_x)), np.float32(float(num_grid_rows) / (max_y - min_y)),
                num_grid_cols, num_grid_rows)


class FrameGeometry(C.Structure):
    """ovs_frame_geometry: what frame::can_observe and the motion model's reprojection read of the current frame."""
    _fields_ = [("camera", Camera), ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("rot_cw", C.c_double * 9), ("trans_cw", C.c_double * 3), ("cam_center", C.c_double * 3),
                ("num_scale_levels", C.c_int32), ("log_scale_factor", C.c_float)]


def _pose12(pose_cw):
    """12 values (R row-major, t) from a 12-vector or a 3x4 / 4x4 cam_pose_cw_"""
    P = np.asarray(pose_cw, np.float64)
    if P.ndim == 2:
        return np.concatenate([P[:3, :3].reshape(9), P[:3, 3]])
    return P.reshape(12)


def frame_geometry(camera, img_bounds, pose_cw, num_scale_levels, log_scale_factor, cam_center=None):
    """camera: optimize.camera(...) (perspective, fisheye and radial_division reproject with the pinhole formula on undistorted
    keypoints); img_bounds = (min_x, max_x, min_y, max_y) (camera_->img_bounds_); pose_cw: 12 values (R row-major, t) or a 3x4 / 4x4
    matrix; cam_center: the frame's cam_center_ (default -R^T t); log_scale_factor: frame::log_scale_factor_ (float)."""
    P = _pose12(pose_cw)
    R, t = P[:9].reshape(3, 3), P[9:]
    if cam_center is None:
        cam_center = -(R.T @ t)
    g = FrameGeometry()
    g.camera = camera
    g.min_x, g.max_x, g.min_y, g.max_y = (float(np.float32(v)) for v in img_bounds)
    g.rot_cw[:] = [float(v) for v in R.reshape(9)]
    g.trans_cw[:] = [float(v) for v in t]
    g.cam_center[:] = [float(v) for v in np.reshape(cam_center, 3)]
    g.num_scale_levels = int(num_scale_levels)
    g.log_scale_factor = float(np.float32(log_scale_factor))
    return g


def _f32(a):
    a = np.ascontiguousarray(a, np.float32)
    return a, a.ctypes.data_as(C.c_void_p)


def _i32(a):
    a = np.ascontiguousarray(a, np.int32)
    return a, a.ctypes.data_as(C.c_void_p)


def _u8p(a):
    if a is None:
        return None, None
    a = np.ascontiguousarray(a, np.uint8)
    return a, a.ctypes.data_as(C.c_void_p)


def _f64(a):
    a = np.ascontiguousarray(a, np.float64)
    return a, a.ctypes.data_as(C.c_void_p)


class frame_index:
    """The matcher-side view of a data::frame: undist_keypts_ (pt, octave, angle), stereo_x_right_,
    descriptors_ and the keypoint grid, resident on the device."""

    def __init__(self, matcher, x, y, octave, angle, x_right, desc, grid):
        self._m = matcher
        x, px = _f32(x); y, py = _f32(y); octave, po = _i32(octave); angle, pa = _f32(angle)
        pxr = None
        if x_right is not None:
            x_right, pxr = _f32(x_right)
        d, pd = _desc(desc)
        self.n = len(x)
        self.grid = grid
        self._h = C.c_void_p()
        _lib.check(_lib.lib().ovs_frame_index_create(matcher._h, self.n, px, py, po, pa, pxr, pd, C.byref(grid), C.byref(self._h)))
        matcher._indexes.add(self._h.value)

    @classmethod
    def from_device(cls, matcher, n, d_keypts_ptr, d_desc_ptr, grid, d_x_right_ptr=None):
        """Index over the device output of orb_extractor.extract_device (keypoint records + descriptors stay on the GPU)."""
        self = cls.__new__(cls)
        self._m = matcher
        self.n = int(n)
        self.grid = grid
        self._h = C.c_void_p()
        _lib.check(_lib.lib().ovs_frame_index_create_device(matcher._h, self.n, C.c_void_p(d_keypts_ptr), C.c_void_p(d_desc_ptr),
                                                             C.c_void_p(d_x_right_ptr) if d_x_right_ptr else None, C.byref(grid), C.byref(self._h)))
        matcher._indexes.add(self._h.value)
        return self

    def close(self):
        if getattr(self, "_h", None):
            live = self._m._indexes
            if self._h.value in live:      # else the matcher was closed first and destroyed this index with it
                live.discard(self._h.value)
                _lib.lib().ovs_frame_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def window_topk(self, ref_xy, margin, min_level, max_level, qdesc, x_right_q=None):
        ref_xy, pr = _f32(ref_xy); margin, pm = _f32(margin); min_level, plo = _i32(min_level); max_level, phi = _i32(max_level)
        q, pq = _desc(qdesc)
        pxr = None
        if x_right_q is not None:
            x_right_q, pxr = _f32(x_right_q)
        nq = len(margin)
        idx = np.zeros((nq, 4), np.int32); dist = np.zeros((nq, 4), np.int32)
        _lib.check(_lib.lib().ovs_match_window_topk_host(self._h, nq, pr, pm, plo, phi, pxr, pq, idx.ctypes.data_as(C.c_void_p),
                                                         dist.ctypes.data_as(C.c_void_p)))
        return idx, dist


def _landmark_arrays(pos_w, mean_normal, min_valid_dist, max_valid_dist):
    pos, pp = _f64(np.reshape(pos_w, (-1, 3))); nrm, pn = _f64(np.reshape(mean_normal, (-1, 3)))
    lo, plo = _f32(min_valid_dist); hi, phi = _f32(max_valid_dist)
    n = len(pos)
    if len(nrm) != n or len(lo) != n or len(hi) != n:
        raise ValueError("one position, mean normal and pair of valid distances per landmark")
    return pos, pp, nrm, pn, lo, plo, hi, phi, n


def _u8n(a, n, what):
    """_u8p of an optional per-item flag array that must have n entries"""
    if a is not None and np.size(a) != n:
        raise ValueError("%s: %d entries, expected %d" % (what, np.size(a), n))
    return _u8p(a)


def _can_observe_outputs(n):
    return (np.zeros(max(n, 1), np.uint8), np.zeros((max(n, 1), 2), np.float32), np.zeros(max(n, 1), np.float32),
            np.zeros(max(n, 1), np.int32))


class projection(_matcher_handle):
    """openvslam::match::projection (lowe_ratio_, check_orientation_)."""

    def __init__(self, lowe_ratio=0.6, check_orientation=True, device=0):
        super().__init__(device)
        self.lowe_ratio_ = float(lowe_ratio)
        self.check_orientation_ = bool(check_orientation)

    def match_frame_and_landmarks(self, frm, scale_factors, reproj_xy, x_right_in_tracking, pred_scale_level, lm_desc,
                                  lm_usable=None, kp_has_observed_lm=None, margin=5.0):
        sf, psf = _f32(scale_factors); rp, prp = _f32(reproj_xy); lv, plv = _i32(pred_scale_level); d, pd = _desc(lm_desc)
        pxr = None
        if x_right_in_tracking is not None:
            x_right_in_tracking, pxr = _f32(x_right_in_tracking)
        _keep5, pu = _u8p(lm_usable); _keep6, pk = _u8p(kp_has_observed_lm)
        out = np.full(max(frm.n, 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_projection_match_frame_and_landmarks_host(frm._h, psf, len(sf), len(lv), pu, prp, pxr, plv, pd, pk, C.c_float(margin),
                                                                            C.c_float(self.lowe_ratio_), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:frm.n]

    def match_current_and_last_frames(self, curr, scale_factors, num_scale_levels, last_usable, reproj_xy, reproj_x_right, last_scale_level,
                                      last_angle, lm_desc, kp_has_observed_lm=None, margin=20.0, assume_forward=False, assume_backward=False):
        sf, psf = _f32(scale_factors); rp, prp = _f32(reproj_xy); lv, plv = _i32(last_scale_level); d, pd = _desc(lm_desc)
        la, pla = _f32(last_angle); lu, plu = _u8p(last_usable)
        pxr = None
        if reproj_x_right is not None:
            reproj_x_right, pxr = _f32(reproj_x_right)
        _keep7, pk = _u8p(kp_has_observed_lm)
        out = np.full(max(curr.n, 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_projection_match_current_and_last_host(curr._h, psf, int(num_scale_levels), len(lv), plu, prp, pxr, plv, pla, pd, pk,
                                                                         C.c_float(margin), int(assume_forward), int(assume_backward),
                                                                         int(self.check_orientation_), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:curr.n]


    def can_observe(self, geometry, pos_w, mean_normal, min_valid_dist, max_valid_dist, ray_cos_thr=0.5, usable=None):
        """frame::can_observe(lm, ray_cos_thr, ...) for every landmark in one launch.  pos_w / mean_normal: (n, 3); min_valid_dist /
        max_valid_dist: the landmarks' raw min_valid_dist_ / max_valid_dist_; usable: the tracker's skip rule (None: all)
        -> observable (n,) bool, reproj_xy (n, 2) f32, x_right (n,) f32, pred_scale_level (n,) i32 (zeros where not observable)."""
        pos, pp, nrm, pn, lo, plo, hi, phi, n = _landmark_arrays(pos_w, mean_normal, min_valid_dist, max_valid_dist)
        _keep, pu = _u8n(usable, n, "usable")
        ok, uv, xr, lv = _can_observe_outputs(n)
        _lib.check(_lib.lib().ovs_frame_can_observe_host(self._h, C.byref(geometry), n, pu, pp, pn, plo, phi, C.c_float(ray_cos_thr),
                                                         *(a.ctypes.data_as(C.c_void_p) for a in (ok, uv, xr, lv))))
        return ok[:n].astype(bool), uv[:n], xr[:n], lv[:n]

    def search_local_landmarks(self, frm, geometry, scale_factors, pos_w, mean_normal, min_valid_dist, max_valid_dist, lm_desc, usable=None,
                               kp_has_observed_lm=None, margin=5.0, ray_cos_thr=0.5):
        """The compute of tracking_module::search_local_landmarks: can_observe on the device, then match_frame_and_landmarks on its
        outputs -> (num_matches, matched_lm_of_kp (frm.n,), observable, reproj_xy, x_right, pred_scale_level)."""
        pos, pp, nrm, pn, lo, plo, hi, phi, n = _landmark_arrays(pos_w, mean_normal, min_valid_dist, max_valid_dist)
        sf, psf = _f32(scale_factors); d, pd = _desc(lm_desc)
        if len(sf) != geometry.num_scale_levels:
            raise ValueError("search_local_landmarks: one scale factor per level")
        if len(d) != n:
            raise ValueError("search_local_landmarks: one descriptor per landmark")
        _keep, pu = _u8n(usable, n, "usable"); _keep2, pk = _u8n(kp_has_observed_lm, frm.n, "kp_has_observed_lm")
        ok, uv, xr, lv = _can_observe_outputs(n)
        out = np.full(max(frm.n, 1), -1, np.int32); nm = C.c_int(0)
        _lib.check(_lib.lib().ovs_projection_search_local_landmarks_host(
            frm._h, C.byref(geometry), psf, n, pu, pp, pn, plo, phi, pd, pk, C.c_float(ray_cos_thr), C.c_float(margin), C.c_float(self.lowe_ratio_),
            *(a.ctypes.data_as(C.c_void_p) for a in (ok, uv, xr, lv, out)), C.byref(nm)))
        return nm.value, out[:frm.n], ok[:n].astype(bool), uv[:n], xr[:n], lv[:n]

    def match_current_and_last_frames_reproject(self, curr, geometry, last_pose_cw, scale_factors, pos_w, last_octave, last_angle, lm_desc,
                                                last_usable=None, kp_has_observed_lm=None, margin=20.0, is_monocular=True, true_baseline=0.0):
        """match_current_and_last_frames(curr_frm, last_frm, margin) with the last frame's landmarks reprojected on the device and the
        direction taken from the two poses -> (num_matches, matched_last_of_kp (curr.n,), in_image (n,) bool, reproj_xy (n, 2))."""
        pos, pp = _f64(np.reshape(pos_w, (-1, 3)))
        n = len(pos)
        sf, psf = _f32(scale_factors); lv, plv = _i32(last_octave); la, pla = _f32(last_angle); d, pd = _desc(lm_desc)
        if len(sf) != geometry.num_scale_levels:
            raise ValueError("match_current_and_last_frames_reproject: one scale factor per level")
        if len(lv) != n or len(la) != n or len(d) != n:
            raise ValueError("match_current_and_last_frames_reproject: one octave, angle and descriptor per last-frame keypoint")
        lp, plp = _f64(_pose12(last_pose_cw))
        _keep, pu = _u8n(last_usable, n, "last_usable"); _keep2, pk = _u8n(kp_has_observed_lm, curr.n, "kp_has_observed_lm")
        ok = np.zeros(max(n, 1), np.uint8); uv = np.zeros((max(n, 1), 2), np.float32)
        out = np.full(max(curr.n, 1), -1, np.int32); nm = C.c_int(0)
        _lib.check(_lib.lib().ovs_projection_match_current_and_last_reproject_host(
            curr._h, C.byref(geometry), int(bool(is_monocular)), C.c_double(true_baseline), plp, psf, n, pu, pp, plv, pla, pd, pk,
            C.c_float(margin), int(self.check_orientation_), out.ctypes.data_as(C.c_void_p), C.byref(nm), ok.ctypes.data_as(C.c_void_p),
            uv.ctypes.data_as(C.c_void_p)))
        return nm.value, out[:curr.n], ok[:n].astype(bool), uv[:n]

    def match_best(self, frm, ref_xy, ref_x_right, margin, min_level, max_level, q_angle, q_desc, usable=None, kp_unavailable=None,
                   hamm_dist_thr=HAMMING_DIST_THR_HIGH):
        """The shared search loop (ovs_projection_match_best_host)."""
        rp, prp = _f32(ref_xy); mg, pmg = _f32(margin); lo, plo = _i32(min_level); hi, phi = _i32(max_level)
        qa, pqa = _f32(q_angle); d, pd = _desc(q_desc)
        pxr = None
        if ref_x_right is not None:
            ref_x_right, pxr = _f32(ref_x_right)
        _keep8, pu = _u8p(usable); _keep9, pk = _u8p(kp_unavailable)
        out = np.full(max(frm.n, 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_projection_match_best_host(frm._h, len(mg), pu, prp, pxr, pmg, plo, phi, pqa, pd, pk, C.c_uint(int(hamm_dist_thr)),
                                                             int(self.check_orientation_), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:frm.n]

    def match_frame_and_keyframe(self, curr, scale_factors, reproj_xy, pred_scale_level, keyfrm_angle, lm_desc, usable, kp_has_lm,
                                 margin, hamm_dist_thr):
        """projection::match_frame_and_keyframe(curr_frm, keyfrm, already_matched_lms, margin, hamm_dist_thr): the caller has
        reprojected the keyframe's landmarks (reproject_to_image, valid-distance test, predict_scale_level -> usable,
        reproj_xy, pred_scale_level); kp_has_lm[i] = curr_frm.landmarks_[i] != nullptr."""
        lvl = np.asarray(pred_scale_level, np.int32)
        sf = np.asarray(scale_factors, np.float32)
        return self.match_best(curr, reproj_xy, None, np.float32(margin) * sf[lvl], lvl - 1, lvl + 1, keyfrm_angle, lm_desc, usable, kp_has_lm,
                               hamm_dist_thr)

    def match_by_Sim3_transform(self, keyfrm, scale_factors, reproj_xy, pred_scale_level, lm_desc, usable, kp_already_matched, margin):
        """projection::match_by_Sim3_transform(keyfrm, Sim3_cw, landmarks, matched_lms_in_keyfrm, margin): landmarks reprojected
        by the caller with the Sim3 pose; window [level-1, level], distance <= HAMMING_DIST_THR_LOW, no orientation check."""
        lvl = np.asarray(pred_scale_level, np.int32)
        sf = np.asarray(scale_factors, np.float32)
        saved, self.check_orientation_ = self.check_orientation_, False
        try:
            return self.match_best(keyfrm, reproj_xy, None, np.float32(margin) * sf[lvl], lvl - 1, lvl, np.zeros(len(lvl), np.float32), lm_desc,
                                   usable, kp_already_matched, HAMMING_DIST_THR_LOW)
        finally:
            self.check_orientation_ = saved


    def match_keyframes_mutually(self, keyfrm_1, keyfrm_2, scale_factors, usable_1, reproj_1_in_2, pred_level_1_in_2, lm_desc_1,
                                 usable_2, reproj_2_in_1, pred_level_2_in_1, lm_desc_2, margin):
        """projection::match_keyframes_mutually: -> (num_matches, matched_idx_2_of_kp_1[n1]); the caller reprojects with the Sim3s."""
        sf, psf = _f32(scale_factors)
        r12, p12 = _f32(reproj_1_in_2); l12, pl12 = _i32(pred_level_1_in_2); d1, pd1 = _desc(lm_desc_1); _keep10, pu1 = _u8p(usable_1)
        r21, p21 = _f32(reproj_2_in_1); l21, pl21 = _i32(pred_level_2_in_1); d2, pd2 = _desc(lm_desc_2); _keep11, pu2 = _u8p(usable_2)
        out = np.full(max(keyfrm_1.n, 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_projection_match_keyframes_mutually_host(keyfrm_1._h, keyfrm_2._h, psf, pu1, p12, pl12, pd1, pu2, p21, pl21, pd2,
                                                                           C.c_float(margin), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:keyfrm_1.n]


class bow_tree(_matcher_handle):
    """openvslam::match::bow_tree (lowe_ratio_, check_orientation_); the BoW node ids of the keypoints are inputs."""

    def __init__(self, lowe_ratio=0.6, check_orientation=True, device=0):
        super().__init__(device)
        self.lowe_ratio_ = float(lowe_ratio)
        self.check_orientation_ = bool(check_orientation)

    def match_frame_and_keyframe(self, desc_kf, angle_kf, lm_valid_kf, bow_node_kf, desc_frm, angle_frm, bow_node_frm):
        """-> (num_matches, matched_keyfrm_idx_of_frm[n_frm])"""
        dk, pdk = _desc(desc_kf); ak, pak = _f32(angle_kf); vk, pvk = _u8p(lm_valid_kf); nk, pnk = _i32(bow_node_kf)
        df, pdf = _desc(desc_frm); af, paf = _f32(angle_frm); nf, pnf = _i32(bow_node_frm)
        out = np.full(max(len(af), 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_bow_tree_match_frame_and_keyframe_host(self._h, len(ak), pdk, pak, pvk, pnk, len(af), pdf, paf, pnf, C.c_float(self.lowe_ratio_),
                                                                         int(self.check_orientation_), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:len(af)]

    def match_keyframes(self, desc_1, angle_1, lm_valid_1, bow_node_1, desc_2, angle_2, lm_valid_2, bow_node_2):
        """-> (num_matches, matched_idx_2_of_1[n1])"""
        d1, pd1 = _desc(desc_1); a1, pa1 = _f32(angle_1); v1, pv1 = _u8p(lm_valid_1); n1, pn1 = _i32(bow_node_1)
        d2, pd2 = _desc(desc_2); a2, pa2 = _f32(angle_2); v2, pv2 = _u8p(lm_valid_2); n2, pn2 = _i32(bow_node_2)
        out = np.full(max(len(a1), 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_bow_tree_match_keyframes_host(self._h, len(a1), pd1, pa1, pv1, pn1, len(a2), pd2, pa2, pv2, pn2, C.c_float(self.lowe_ratio_),
                                                                int(self.check_orientation_), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:len(a1)]


class FuseTarget(C.Structure):
    """ovs_fuse_target: what match::fuse::replace_duplication reads of one target keyframe."""
    _fields_ = [("geometry", FrameGeometry), ("scale_factors", C.c_void_p), ("inv_level_sigma_sq", C.c_void_p), ("num_keypts", C.c_int32),
                ("x", C.c_void_p), ("y", C.c_void_p), ("octave", C.c_void_p), ("x_right", C.c_void_p), ("descriptors", C.c_void_p),
                ("grid", Grid)]


class fuse_target:
    """One target keyframe of fuse.replace_duplication: its frame_geometry, scale_factors_ and inv_level_sigma_sq_, undist_keypts_
    (x, y, octave), descriptors_ (n, 32), the camera grid and stereo_x_right_ (None: monocular).  Holds the arrays the struct
    points at."""

    def __init__(self, geometry, scale_factors, inv_level_sigma_sq, x, y, octave, desc, grid, x_right=None):
        self.scale_factors, psf = _f32(scale_factors); self.inv_level_sigma_sq, piw = _f32(inv_level_sigma_sq)
        self.x, px = _f32(x); self.y, py = _f32(y); self.octave, po = _i32(octave); self.desc, pd = _desc(desc)
        n = len(self.x)
        if len(self.y) != n or len(self.octave) != n or len(self.desc) != n:
            raise ValueError("fuse_target: one y, octave and descriptor per keypoint")
        if len(self.scale_factors) != geometry.num_scale_levels or len(self.inv_level_sigma_sq) != geometry.num_scale_levels:
            raise ValueError("fuse_target: one scale factor and one inverse sigma^2 per level of the geometry")
        pxr = None
        self.x_right = None
        if x_right is not None:
            self.x_right, pxr = _f32(x_right)
            if len(self.x_right) != n:
                raise ValueError("fuse_target: one x_right per keypoint")
        self.n = n
        self.c = FuseTarget(geometry, psf, piw, n, px, py, po, pxr, pd, grid)


class fuse(_matcher_handle):
    """openvslam::match::fuse: the matching core (best keypoint per reprojected landmark), and replace_duplication's compute for
    many target keyframes at once."""

    def replace_duplication(self, targets, pos_w, mean_normal, min_valid_dist, max_valid_dist, lm_desc, q_off, q_lm, margin=3.0, geometry=False):
        """ovs_fuse_replace_duplication_host: targets = [fuse_target]; landmark table (nlm rows): pos_w / mean_normal (nlm, 3), the raw
        min_valid_dist_ / max_valid_dist_, lm_desc (nlm, 32); the queries of target t are q_lm[q_off[t]:q_off[t + 1]] (a landmark
        row, or -1 to skip) -> (num_fused, best_idx (Q,)), and with geometry=True also passed (Q,) bool, reproj_xy (Q, 2) f32,
        x_right (Q,) f32, pred_level (Q,) i32 (zeros where not passed)."""
        pos, pp, nrm, pn, lo, plo, hi, phi, nlm = _landmark_arrays(pos_w, mean_normal, min_valid_dist, max_valid_dist)
        d, pd = _desc(lm_desc)
        if len(d) != nlm:
            raise ValueError("replace_duplication: one descriptor per landmark")
        B = len(targets)
        arr = (FuseTarget * max(B, 1))(*[t.c for t in targets])
        qo, pqo = _i32(q_off); ql, pql = _i32(q_lm)
        if len(qo) != B + 1:
            raise ValueError("replace_duplication: q_off needs B + 1 entries")
        Q = len(ql)
        if qo[-1] != Q:
            raise ValueError("replace_duplication: q_off[-1] must be len(q_lm)")
        n1 = max(Q, 1)
        best = np.full(n1, -1, np.int32); n = C.c_int(0)
        outs = (np.zeros(n1, np.uint8), np.zeros((n1, 2), np.float32), np.zeros(n1, np.float32), np.zeros(n1, np.int32)) if geometry else None
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(_lib.lib().ovs_fuse_replace_duplication_host(self._h, B, arr, nlm, pp, pn, plo, phi, pd, pqo, pql, C.c_float(margin), vp(best),
                                                                C.byref(n), *((vp(a) for a in outs) if geometry else (None,) * 4)))
        if not geometry:
            return n.value, best[:Q]
        return n.value, best[:Q], outs[0][:Q].astype(bool), outs[1][:Q], outs[2][:Q], outs[3][:Q]

    def best_keypoints(self, keyfrm, reproj_xy, reproj_x_right, pred_level, lm_desc, scale_factors, inv_level_sigma_sq, margin, usable=None):
        rp, prp = _f32(reproj_xy); lv, plv = _i32(pred_level); d, pd = _desc(lm_desc); sf, psf = _f32(scale_factors); iw, piw = _f32(inv_level_sigma_sq)
        pxr = None
        if reproj_x_right is not None:
            reproj_x_right, pxr = _f32(reproj_x_right)
        _keep, pu = _u8p(usable)
        out = np.full(max(len(lv), 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_fuse_best_keypoints_host(keyfrm._h, len(lv), pu, prp, pxr, plv, pd, psf, piw, len(sf), C.c_float(margin),
                                                           out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return n.value, out[:len(lv)]


class area(_matcher_handle):
    """openvslam::match::area (lowe_ratio_, check_orientation_)."""

    def __init__(self, lowe_ratio=0.9, check_orientation=True, device=0):
        super().__init__(device)
        self.lowe_ratio_ = float(lowe_ratio)
        self.check_orientation_ = bool(check_orientation)

    def match_in_consistent_area(self, frm_2, octave_1, angle_1, desc_1, prev_matched_pts, margin=100):
        o1, po = _i32(octave_1); a1, pa = _f32(angle_1); d1, pd = _desc(desc_1)
        prev = np.ascontiguousarray(prev_matched_pts, np.float32).copy()
        n1 = len(o1)
        out = np.full(max(n1, 1), -1, np.int32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_area_match_in_consistent_area_host(frm_2._h, n1, po, pa, pd, prev.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                                                                     int(margin), C.c_float(self.lowe_ratio_), int(self.check_orientation_), C.byref(n)))
        return n.value, out[:n1], prev


class stereo(_matcher_handle):
    """openvslam::match::stereo: built from the two extractors' pyramids, keypoints and descriptors."""

    def compute(self, extractor_left, extractor_right, kps_left, desc_left, kps_right, desc_right, focal_x_baseline, true_baseline):
        lx, plx = _f32(kps_left["x"]); ly, ply = _f32(kps_left["y"]); lo, plo = _i32(kps_left["octave"]); ld, pld = _desc(desc_left)
        rx, prx = _f32(kps_right["x"]); ry, pry = _f32(kps_right["y"]); ro, pro = _i32(kps_right["octave"]); rd, prd = _desc(desc_right)
        nl, nr = len(lx), len(rx)
        xr = np.full(max(nl, 1), -1, np.float32); dp = np.full(max(nl, 1), -1, np.float32); n = C.c_int(0)
        _lib.check(_lib.lib().ovs_stereo_compute_host(self._h, extractor_left._h, extractor_right._h, nl, plx, ply, plo, pld, nr, prx, pry, pro, prd,
                                                      C.c_float(focal_x_baseline), C.c_float(true_baseline), xr.ctypes.data_as(C.c_void_p),
                                                      dp.ctypes.data_as(C.c_void_p), C.byref(n)))
        return xr[:nl], dp[:nl], n.value
