#!/usr/bin/env python
"""Generates tests/golden/rectify_golden.npz: cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap (CV_32FC1)
maps of seeded stereo rigs at small sizes, and cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of seeded u8 images with 1, 3 and
4 channels through them and through edge-case maps (ties, NaN, +-inf, +-FLT_MAX, values outside int), computed with the cv2
wheel of this image.  The rectification oracle is pinned against these vectors by tests/test_rectify_oracle.py.
Re-run: python tests/golden/make_rectify_golden.py"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rectify_cases as RC  # noqa: E402


def cv_maps(model, cols, rows, K, D, R, K_rect):
    if model == "perspective":
        return cv2.initUndistortRectifyMap(K, D, R, K_rect, (cols, rows), cv2.CV_32FC1)
    return cv2.fisheye.initUndistortRectifyMap(K, D, R, K_rect, (cols, rows), cv2.CV_32FC1)


def main():
    out = {"cv2_version": np.array(cv2.__version__)}
    for ci, (model, cols, rows, seed) in enumerate(RC.GOLDEN_CASES):
        r = RC.rig(model, cols, rows, seed, rot=0.1)
        for k, v in r.items():
            out["c%d_%s" % (ci, k)] = v
        for s, side in enumerate(("l", "r")):
            mx, my = cv_maps(model, cols, rows, r["K_" + side], r["D_" + side], r["R_" + side], r["K_rect"])
            out["c%d_map%d_x" % (ci, s)] = mx; out["c%d_map%d_y" % (ci, s)] = my
            for ch in (1, 3, 4):
                img = RC.image(cols, rows, ch, seed * 10 + ch)
                out["c%d_img%d_%d" % (ci, s, ch)] = img
                out["c%d_out%d_%d" % (ci, s, ch)] = cv2.remap(img, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    mx, my = RC.edge_maps(29, 17, 5)
    out["edge_map_x"] = mx; out["edge_map_y"] = my
    for ch in (1, 3, 4):
        img = RC.image(29, 17, ch, 50 + ch)
        out["edge_img_%d" % ch] = img
        out["edge_out_%d" % ch] = cv2.remap(img, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    path = os.path.join(ROOT, "tests", "golden", "rectify_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
