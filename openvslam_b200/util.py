"""Host-side mirror of openvslam::util::stereo_rectifier (src/openvslam/util/stereo_rectifier.{h,cc}), calling the C ABI of
libovs_b200.so.  The maps are built once on the device; rectify() remaps both images there."""
import ctypes as C

import numpy as np

from . import _lib

MODELS = {"perspective": 0, "fisheye": 2}   # OVS_CAMERA_PERSPECTIVE, OVS_CAMERA_FISHEYE
DIST_LEN = {"perspective": 5, "fisheye": 4}


def _mat(a, shape):
    a = np.ascontiguousarray(a, np.float64)
    if a.size != int(np.prod(shape)):
        raise ValueError("expected %s values, got %d" % ("x".join(map(str, shape)), a.size))
    return a


class stereo_rectifier:
    """util::stereo_rectifier from the StereoRectifier block (K_left, D_left, R_left, K_right, D_right, R_right, model) and the
    camera's cols, rows and K (the rectified camera matrix).  D is (k1, k2, p1, p2, k3) for "perspective", (k1..k4) for "fisheye"."""

    def __init__(self, cols, rows, K_rect, K_left, D_left, R_left, K_right, D_right, R_right, model="perspective", device=0):
        if model not in MODELS:
            raise ValueError("model must be perspective or fisheye, got %r" % (model,))
        self.cols, self.rows, self.model = int(cols), int(rows), model
        nd = DIST_LEN[model]
        arrs = [_mat(K_left, (3, 3)), _mat(D_left, (nd,)), _mat(R_left, (3, 3)), _mat(K_right, (3, 3)), _mat(D_right, (nd,)),
                _mat(R_right, (3, 3)), _mat(K_rect, (3, 3))]
        self._h = C.c_void_p()
        _lib.check(_lib.lib().ovs_stereo_rectifier_create(int(device), MODELS[model], self.cols, self.rows,
                                                          *[a.ctypes.data_as(C.c_void_p) for a in arrs], C.byref(self._h)))

    @property
    def handle(self):
        return self._h

    def close(self):
        if getattr(self, "_h", None):
            _lib.lib().ovs_stereo_rectifier_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def maps(self, side):
        """(map_x, map_y) of side 0 (left) or 1 (right): rows x cols float32, as cv::initUndistortRectifyMap returns them."""
        mx = np.empty((self.rows, self.cols), np.float32); my = np.empty((self.rows, self.cols), np.float32)
        _lib.check(_lib.lib().ovs_stereo_rectifier_maps(self._h, int(side), mx.ctypes.data_as(C.c_void_p), my.ctypes.data_as(C.c_void_p)))
        return mx, my

    def rectify(self, in_img_l, in_img_r):
        """rectify(in_img_l, in_img_r) -> (out_img_l, out_img_r): u8 H x W or H x W x {3, 4}, channels kept."""
        l = np.ascontiguousarray(in_img_l, np.uint8); r = np.ascontiguousarray(in_img_r, np.uint8)
        if l.shape != r.shape or l.ndim not in (2, 3):
            raise ValueError("left and right images must have the same shape, H x W or H x W x C")
        ch = 1 if l.ndim == 2 else l.shape[2]
        out_l = np.empty_like(l); out_r = np.empty_like(r)
        _lib.check(_lib.lib().ovs_stereo_rectify_host(self._h, l.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p), l.shape[1],
                                                      l.shape[0], C.c_size_t(l.strides[0]), ch, out_l.ctypes.data_as(C.c_void_p),
                                                      out_r.ctypes.data_as(C.c_void_p), C.c_size_t(out_l.strides[0])))
        return out_l, out_r
