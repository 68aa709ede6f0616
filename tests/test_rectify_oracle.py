"""The stereo rectification oracle (oracle/rectify_oracle.c) against OpenCV: the perspective map bit for bit and the fisheye map
within one float ulp (atan), remap INTER_LINEAR / BORDER_CONSTANT bit for bit for 1, 3 and 4 channels -- live against the cv2
wheel and against the committed fixture tests/golden/rectify_golden.npz."""
import os

import numpy as np
import pytest

import rectify_cases as RC

cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rectify_golden.npz")


@pytest.fixture(scope="module")
def RO(oracle):
    from oracle import rectify
    return rectify


def _cv_maps(model, cols, rows, K, D, R, K_rect):
    if model == "perspective":
        return cv2.initUndistortRectifyMap(K, D, R, K_rect, (cols, rows), cv2.CV_32FC1)
    return cv2.fisheye.initUndistortRectifyMap(K, D, R, K_rect, (cols, rows), cv2.CV_32FC1)


def _cv_remap(img, mx, my):
    return cv2.remap(img, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


@pytest.mark.parametrize("model", ["perspective", "fisheye"])
@pytest.mark.parametrize("cols,rows", RC.SIZES)
def test_maps_and_remap_equal_cv2(RO, model, cols, rows):
    r = RC.rig(model, cols, rows, seed=cols * 7 + rows, rot=0.1)
    differing = 0
    for side in ("l", "r"):
        args = (r["K_" + side], r["D_" + side], r["R_" + side], r["K_rect"])
        cx, cy = _cv_maps(model, cols, rows, *args)
        ox, oy = RO.init_rectify_map(model, cols, rows, *args)
        d = np.maximum(RC.ulp_distance(ox, cx), RC.ulp_distance(oy, cy))
        if model == "perspective":
            assert d.max() == 0, "perspective map: %d entries differ" % int((d > 0).sum())
        else:
            assert d.max() <= 1, "fisheye map: %d entries differ, up to %d ulp" % (int((d > 0).sum()), int(d.max()))
        differing += int((d > 0).sum())
        inside = (cx >= 0) & (cx <= cols - 1) & (cy >= 0) & (cy <= rows - 1)
        if cols * rows > 100:
            assert 0.5 < inside.mean() < 1.0, "the rig's maps should fall partly outside the image"
        for ch in (1, 3, 4):
            img = RC.image(cols, rows, ch, seed=cols + rows + ch)
            assert np.array_equal(RO.remap(img, cx, cy), _cv_remap(img, cx, cy)), ch
    print("%s %dx%d: %d map entries differ from cv2 by one ulp" % (model, cols, rows, differing))


@pytest.mark.parametrize("model", ["perspective", "fisheye"])
def test_strong_rotation_maps(RO, model):
    # rotations of up to ~90 degrees: rays behind the camera (fisheye: -+inf), NaN-free huge perspective projections
    cols, rows = 160, 120
    for seed in range(4):
        r = RC.rig(model, cols, rows, seed=100 + seed, rot=1.2)
        for side in ("l", "r"):
            args = (r["K_" + side], r["D_" + side], r["R_" + side], r["K_rect"])
            cx, cy = _cv_maps(model, cols, rows, *args)
            ox, oy = RO.init_rectify_map(model, cols, rows, *args)
            d = np.maximum(RC.ulp_distance(ox, cx), RC.ulp_distance(oy, cy))
            assert d.max() <= (0 if model == "perspective" else 1)
            img = RC.image(cols, rows, 3, seed)
            assert np.array_equal(RO.remap(img, cx, cy), _cv_remap(img, cx, cy))


@pytest.mark.parametrize("cols,rows", [(1, 1), (7, 5), (29, 17), (333, 97)])
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_edge_maps(RO, cols, rows, channels):
    mx, my = RC.edge_maps(cols, rows, seed=cols * rows)
    img = RC.image(cols, rows, channels, seed=channels)
    assert np.array_equal(RO.remap(img, mx, my), _cv_remap(img, mx, my))


def test_remap_fully_outside_and_ties(RO):
    img = RC.image(40, 30, 3, seed=1)
    far = np.full((30, 40), 1e5, np.float32)
    assert not RO.remap(img, far, far).any() and not _cv_remap(img, far, far).any()
    # every tie k + (2m + 1)/64 along a row: cvRound rounds half to even
    xs = (3 + np.arange(64, dtype=np.float32) / 64).reshape(1, 64).repeat(3, 0)
    ys = np.full_like(xs, 1.5 + 1.0 / 64)
    g = RC.image(10, 4, 1, seed=2)
    assert np.array_equal(RO.remap(g, xs, ys), _cv_remap(g, xs, ys))
    q = RO.quantise(np.array([0.5 / 32, 1.5 / 32, 2.5 / 32, np.nan, np.inf, -np.inf, 1e9, -1e9], np.float32))
    assert q.tolist() == [0, 2, 2] + [-2 ** 31] * 5


@pytest.mark.parametrize("cols,rows", [(7, 5), (752, 480)])
def test_identity_rectification(RO, cols, rows):
    # perspective only: the fisheye model with zero coefficients still maps a pinhole ray through atan
    r = RC.identity_rig("perspective", cols, rows)
    mx, my = RO.init_rectify_map("perspective", cols, rows, r["K_l"], r["D_l"], r["R_l"], r["K_rect"])
    jj, ii = np.meshgrid(np.arange(cols, dtype=np.float32), np.arange(rows, dtype=np.float32))
    assert np.array_equal(mx, jj) and np.array_equal(my, ii)
    for ch in (1, 3, 4):
        img = RC.image(cols, rows, ch, seed=ch)
        assert np.array_equal(RO.remap(img, mx, my), img)


def test_golden_fixture(RO):
    g = np.load(GOLDEN)
    for ci, (model, cols, rows, _) in enumerate(RC.GOLDEN_CASES):
        for s, side in enumerate(("l", "r")):
            ox, oy = RO.init_rectify_map(model, cols, rows, g["c%d_K_%s" % (ci, side)], g["c%d_D_%s" % (ci, side)],
                                         g["c%d_R_%s" % (ci, side)], g["c%d_K_rect" % ci])
            gx, gy = g["c%d_map%d_x" % (ci, s)], g["c%d_map%d_y" % (ci, s)]
            d = np.maximum(RC.ulp_distance(ox, gx), RC.ulp_distance(oy, gy))
            assert d.max() <= (0 if model == "perspective" else 1), (ci, s)
            for ch in (1, 3, 4):
                assert np.array_equal(RO.remap(g["c%d_img%d_%d" % (ci, s, ch)], gx, gy), g["c%d_out%d_%d" % (ci, s, ch)]), (ci, s, ch)
    for ch in (1, 3, 4):
        assert np.array_equal(RO.remap(g["edge_img_%d" % ch], g["edge_map_x"], g["edge_map_y"]), g["edge_out_%d" % ch]), ch
