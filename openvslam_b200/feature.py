"""Host-side mirror of openvslam::feature::{orb_params, orb_extractor}
(src/openvslam/feature/orb_params.h, orb_extractor.h -- names as recalled in SURVEY.md 8a),
calling the C ABI of libovs_b200.so.  Same member names and argument meaning as the reference."""
import ctypes as C
import numpy as np

from . import _lib

# cv::KeyPoint, 28 bytes
KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"),
                           ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])
assert KEYPOINT_DTYPE.itemsize == 28


class orb_params:
    """openvslam::feature::orb_params: max_num_keypts_, scale_factor_, num_levels_,
    ini_fast_thr_, min_fast_thr, mask_rects_ ({x_min, x_max, y_min, y_max} in [0,1])."""

    def __init__(self, max_num_keypts=2000, scale_factor=1.2, num_levels=8, ini_fast_thr=20, min_fast_thr=7,
                 mask_rects=()):
        self.max_num_keypts_ = int(max_num_keypts)
        self.scale_factor_ = float(scale_factor)
        self.num_levels_ = int(num_levels)
        self.ini_fast_thr_ = int(ini_fast_thr)
        self.min_fast_thr = int(min_fast_thr)
        self.mask_rects_ = [list(map(float, r)) for r in mask_rects]
        for r in self.mask_rects_:
            if len(r) != 4:
                raise ValueError("Each of mask rectangles must contain four parameters")
            if r[0] >= r[1] or r[2] >= r[3]:
                raise ValueError("x_max/y_max must be greater than x_min/y_min")


class orb_extractor:
    """openvslam::feature::orb_extractor.  extract(image, mask) -> (keypts, descriptors)."""

    def __init__(self, params=None, device=0, **kw):
        self.orb_params_ = params if params is not None else orb_params(**kw)
        p = self.orb_params_
        cp = _lib.OrbParams(p.max_num_keypts_, p.scale_factor_, p.num_levels_, p.ini_fast_thr_, p.min_fast_thr)
        rects = np.ascontiguousarray(p.mask_rects_, np.float32).reshape(-1, 4)
        self._h = C.c_void_p()
        _lib.check(_lib.lib().ovs_extractor_create(C.byref(cp), rects.ctypes.data_as(C.c_void_p) if len(rects) else None,
                                                   len(rects), int(device), C.byref(self._h)))
        self._cap = _lib.lib().ovs_extractor_max_keypoints(self._h)
        self._kps = np.zeros(self._cap, KEYPOINT_DTYPE)
        self._desc = np.zeros((self._cap, 32), np.uint8)
        L = p.num_levels_
        self.scale_factors_ = np.zeros(L, np.float32); self.inv_scale_factors_ = np.zeros(L, np.float32)
        self.level_sigma_sq_ = np.zeros(L, np.float32); self.inv_level_sigma_sq_ = np.zeros(L, np.float32)
        _lib.check(_lib.lib().ovs_extractor_scale_factors(self._h, *[a.ctypes.data_as(C.c_void_p) for a in (
            self.scale_factors_, self.inv_scale_factors_, self.level_sigma_sq_, self.inv_level_sigma_sq_)]))

    def close(self):
        if getattr(self, "_h", None):
            _lib.lib().ovs_extractor_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- orb_extractor::extract(in_image, in_image_mask, keypts, out_descriptors)
    def extract(self, image, mask=None, color_order="BGR", rectifier=None, side=0):
        """image: H x W (gray) or H x W x {3, 4} u8 (colour: converted like util::convert_to_grayscale with `color_order`).
        rectifier: a util.stereo_rectifier; the raw image of `side` (0 left, 1 right) is rectified on the device first, as
        util::stereo_rectifier::rectify does before the stereo frame is built.  The mask is in rectified coordinates."""
        image = np.asarray(image)
        if image.size == 0:
            return np.zeros(0, KEYPOINT_DTYPE), np.zeros((0, 32), np.uint8)
        color = image.ndim == 3
        if rectifier is not None:
            assert image.dtype == np.uint8 and (image.ndim == 2 or image.shape[2] in (1, 3, 4)), "image must be CV_8UC1 / 3 / 4"
            image = np.ascontiguousarray(image)
        elif color:
            assert image.dtype == np.uint8 and image.shape[2] in (3, 4), "colour image must be CV_8UC3 / CV_8UC4"
            image = np.ascontiguousarray(image)
        else:
            assert image.dtype == np.uint8 and image.ndim == 2, "image must be CV_8UC1"
            if image.strides[1] != 1:
                image = np.ascontiguousarray(image)
        mp, ms = None, 0
        if mask is not None:
            mask = np.asarray(mask)
            assert mask.dtype == np.uint8 and mask.shape == image.shape[:2], "mask must be CV_8UC1 of the image size"
            if mask.strides[1] != 1:
                mask = np.ascontiguousarray(mask)
            mp, ms = mask.ctypes.data_as(C.c_void_p), mask.strides[0]
        n = C.c_int(0)

        def call():
            if rectifier is not None:
                return _lib.lib().ovs_extract_host_rectified(self._h, rectifier.handle, int(side), image.ctypes.data_as(C.c_void_p),
                                                             image.shape[1], image.shape[0], C.c_size_t(image.strides[0]),
                                                             1 if image.ndim == 2 else image.shape[2],
                                                             1 if color_order.upper().startswith("RGB") else 0, mp, C.c_size_t(ms),
                                                             self._kps.ctypes.data_as(C.c_void_p), self._desc.ctypes.data_as(C.c_void_p),
                                                             self._cap, C.byref(n))
            if color:
                return _lib.lib().ovs_extract_host_color(self._h, image.ctypes.data_as(C.c_void_p), image.shape[1], image.shape[0],
                                                         C.c_size_t(image.strides[0]), image.shape[2], 1 if color_order.upper().startswith("RGB") else 0,
                                                         mp, C.c_size_t(ms), self._kps.ctypes.data_as(C.c_void_p),
                                                         self._desc.ctypes.data_as(C.c_void_p), self._cap, C.byref(n))
            return _lib.lib().ovs_extract_host(self._h, image.ctypes.data_as(C.c_void_p), image.shape[1], image.shape[0],
                                               C.c_size_t(image.strides[0]), mp, C.c_size_t(ms),
                                               self._kps.ctypes.data_as(C.c_void_p), self._desc.ctypes.data_as(C.c_void_p),
                                               self._cap, C.byref(n))
        rc = call()
        if rc == -4:   # OVS_ERR_CAPACITY: a very wide / tall image made the handle grow its keypoint budget (aspect-ratio bound of the tree)
            cap = _lib.lib().ovs_extractor_max_keypoints(self._h)
            if cap > self._cap:
                self._cap = cap
                self._kps = np.zeros(cap, KEYPOINT_DTYPE); self._desc = np.zeros((cap, 32), np.uint8)
                rc = call()
        _lib.check(rc)
        return self._kps[:n.value].copy(), self._desc[:n.value].copy()

    def extract_device(self, d_image_ptr, width, height, pitch, d_kps_ptr, d_desc_ptr, capacity, mask=None):
        """Device-resident variant: raw device pointers in, number of keypoints out."""
        mp, ms = None, 0
        if mask is not None:
            mask = np.ascontiguousarray(mask, np.uint8)
            mp, ms = mask.ctypes.data_as(C.c_void_p), mask.strides[0]
        n = C.c_int(0)
        _lib.check(_lib.lib().ovs_extract_device(self._h, C.c_void_p(d_image_ptr), int(width), int(height), C.c_size_t(pitch),
                                                 mp, C.c_size_t(ms), C.c_void_p(d_kps_ptr), C.c_void_p(d_desc_ptr),
                                                 int(capacity), C.byref(n)))
        return n.value

    # -- data::frame ctor: camera->undistort_keypoints + camera->convert_keypoints_to_bearings
    def undistort_keypoints(self, keypts, cam, dist=None, num_iterations=20):
        """-> (undist_keypts, bearings[n, 3] f64).  cam: optimize.camera(...); dist = (k1, k2, p1, p2, k3) or None."""
        keypts = np.ascontiguousarray(keypts, KEYPOINT_DTYPE)
        n = len(keypts)
        und = np.zeros(n, KEYPOINT_DTYPE); bear = np.zeros((n, 3), np.float64)
        dp = None
        if dist is not None:
            dist = np.ascontiguousarray(dist, np.float64)
            want = {0: 5, 2: 4, 3: 1}.get(int(cam.model), 5)
            assert dist.size == want, "dist = (k1, k2, p1, p2, k3) perspective | (k1, k2, k3, k4) fisheye | (distortion,) radial division"
            dp = dist.ctypes.data_as(C.c_void_p)
        _lib.check(_lib.lib().ovs_undistort_keypoints_host(self._h, C.byref(cam), dp, int(num_iterations), n, keypts.ctypes.data_as(C.c_void_p),
                                                           und.ctypes.data_as(C.c_void_p), bear.ctypes.data_as(C.c_void_p)))
        return und, bear

    # -- orb_extractor::image_pyramid_
    def image_pyramid(self, level):
        w, h = C.c_int(), C.c_int()
        _lib.check(_lib.lib().ovs_extractor_pyramid_level(self._h, level, None, None, C.byref(w), C.byref(h)))
        out = np.empty((h.value, w.value), np.uint8)
        _lib.check(_lib.lib().ovs_extractor_copy_pyramid_level(self._h, level, out.ctypes.data_as(C.c_void_p), C.c_size_t(w.value)))
        return out

    def pyramid_level_device(self, level):
        ptr, pitch, w, h = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
        _lib.check(_lib.lib().ovs_extractor_pyramid_level(self._h, level, C.byref(ptr), C.byref(pitch), C.byref(w), C.byref(h)))
        return ptr.value, pitch.value, w.value, h.value

    # -- stage taps used by the parity tests
    def debug_score_map(self, level):
        _, _, w, h = self.pyramid_level_device(level)
        out = np.empty((h, w), np.uint8)
        _lib.check(_lib.lib().ovs_extractor_debug_score_map(self._h, level, out.ctypes.data_as(C.c_void_p), C.c_size_t(w)))
        return out

    def debug_candidates(self, level):
        n = C.c_int(0)
        _lib.check(_lib.lib().ovs_extractor_debug_candidates(self._h, level, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), 3), np.int32)
        _lib.check(_lib.lib().ovs_extractor_debug_candidates(self._h, level, out.ctypes.data_as(C.c_void_p), n.value, C.byref(n)))
        return out[:n.value]

    def last_timings_us(self):
        t = np.zeros(8, np.float32)
        _lib.check(_lib.lib().ovs_extractor_last_timings(self._h, t.ctypes.data_as(C.c_void_p)))
        return dict(zip(("upload", "pyramid", "fast_score", "cell_nms_compact", "tree_distribute", "orient_describe", "download", "total_wall"),
                        map(float, t)))
