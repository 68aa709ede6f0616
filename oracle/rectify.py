"""ctypes front for the stereo rectification oracle (oracle/rectify_oracle.c, built into oracle/liboracle.so with the rest of the
oracle).  TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/; the product package never imports this module.
Camera matrices are 3 x 3 float64; dist is (k1, k2, p1, p2, k3) for model "perspective" and (k1, k2, k3, k4) for "fisheye"."""
import ctypes as C

import numpy as np

from .oracle import lib

MODELS = {"perspective": 0, "fisheye": 2}
DIST_LEN = {"perspective": 5, "fisheye": 4}


def _p(a, dt):
    a = np.ascontiguousarray(a, dt)
    return a, a.ctypes.data_as(C.c_void_p)


def rectify_inverse(K_rect, R):
    """(K_rect R)^-1 as initUndistortRectifyMap forms it."""
    K_rect, pk = _p(K_rect, np.float64); R, pr = _p(R, np.float64)
    out = np.zeros((3, 3), np.float64)
    assert lib().orc_rectify_inverse(pk, pr, out.ctypes.data_as(C.c_void_p)), "K_rect R is singular"
    return out


def init_rectify_map(model, cols, rows, K, dist, R, K_rect):
    """cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap with CV_32FC1 maps -> (map_x, map_y) rows x cols f32."""
    K, pk = _p(K, np.float64); R, pr = _p(R, np.float64); K_rect, pkr = _p(K_rect, np.float64)
    dist, pd = _p(np.reshape(dist, -1), np.float64)
    assert dist.size == DIST_LEN[model], "dist has %d coefficients for the %s model" % (DIST_LEN[model], model)
    mx = np.zeros((rows, cols), np.float32); my = np.zeros((rows, cols), np.float32)
    ok = lib().orc_init_rectify_map(MODELS[model], int(cols), int(rows), pk, pd, pr, pkr, mx.ctypes.data_as(C.c_void_p),
                                    my.ctypes.data_as(C.c_void_p))
    assert ok, "K_rect R is singular"
    return mx, my


def remap(img, map_x, map_y):
    """cv::remap(img, map_x, map_y, INTER_LINEAR, BORDER_CONSTANT, 0): H x W or H x W x {1, 3, 4} u8 -> map-sized image."""
    img = np.ascontiguousarray(img, np.uint8)
    c = 1 if img.ndim == 2 else img.shape[2]
    assert c in (1, 3, 4)
    map_x, px = _p(map_x, np.float32); map_y, py = _p(map_y, np.float32)
    assert map_x.shape == map_y.shape and map_x.ndim == 2
    mh, mw = map_x.shape
    out = np.zeros((mh, mw) + img.shape[2:], np.uint8)
    lib().orc_remap_linear(img.ctypes.data_as(C.c_void_p), img.shape[1], img.shape[0], img.strides[0], c, px, py, mw, mh,
                           out.ctypes.data_as(C.c_void_p), out.strides[0])
    return out


def quantise(m):
    """The fixed-point map entries remap uses: cvRound(m * 32) per entry, INT_MIN for NaN and out-of-range products."""
    m = np.ascontiguousarray(m, np.float32).ravel()
    f = lib().orc_remap_quantise
    f.restype = C.c_int; f.argtypes = [C.c_float]
    return np.array([f(float(v)) for v in m], np.int32)


def rectify(model, K_l, D_l, R_l, K_r, D_r, R_r, K_rect, img_l, img_r):
    """util::stereo_rectifier::rectify: both images through their own maps."""
    h, w = np.asarray(img_l).shape[:2]
    ml = init_rectify_map(model, w, h, K_l, D_l, R_l, K_rect)
    mr = init_rectify_map(model, w, h, K_r, D_r, R_r, K_rect)
    return remap(img_l, *ml), remap(img_r, *mr)
