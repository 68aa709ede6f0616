"""Vectorised numpy restatement of the tracker's per-landmark geometry (camera::reproject_to_image, frame::can_observe,
landmark::predict_scale_level, the motion model's direction), with the summation orders of DESIGN.md section 5.  It pins the C
oracle (oracle/tracking_oracle.c) on the CPU.  The transcendental functions go through Python's math module (the C library), one
element at a time, so that no vectorised log / asin / atan2 of numpy's own stands in for the C library's."""
import math

import numpy as np

_asin = np.frompyfunc(math.asin, 1, 1)
_atan2 = np.frompyfunc(math.atan2, 2, 1)


def _libm(f, *a):
    return np.asarray(f(*a), np.float64).reshape(np.shape(a[0]))


def _rows(g):
    R = np.array(g.rot_cw[:], np.float64).reshape(3, 3)
    t = np.array(g.trans_cw[:], np.float64)
    return R, t


def reproject(g, pos_w, usable=None):
    """-> in_image (n,) bool, reproj_xy (n, 2) f32, x_right (n,) f32 (zeros where not in the image)"""
    P = np.asarray(pos_w, np.float64).reshape(-1, 3)
    n = len(P)
    R, t = _rows(g)
    with np.errstate(all="ignore"):
        # each row: ((r0 x + r1 y) + r2 z) + t
        pc = np.stack([((R[r, 0] * P[:, 0] + R[r, 1] * P[:, 1]) + R[r, 2] * P[:, 2]) + t[r] for r in range(3)], 1)
        c = g.camera
        if c.model == 1:
            L = np.sqrt((pc[:, 0] * pc[:, 0] + pc[:, 1] * pc[:, 1]) + pc[:, 2] * pc[:, 2])
            bx, by, bz = pc[:, 0] / L, pc[:, 1] / L, pc[:, 2] / L
            lat = -_libm(_asin, by)
            lon = _libm(_atan2, bx, bz)
            u = c.cols * (0.5 + lon / (2.0 * math.pi))
            v = c.rows * (0.5 - lat / math.pi)
            xr = np.full(n, -1.0, np.float32)
            ok = np.ones(n, bool)
        else:
            front = ~(pc[:, 2] <= 0.0)
            z_inv = 1.0 / pc[:, 2]
            u = (c.fx * pc[:, 0]) * z_inv + c.cx
            v = (c.fy * pc[:, 1]) * z_inv + c.cy
            xr = (u - c.focal_x_baseline * z_inv).astype(np.float32)
            inside = ~((u < np.float64(np.float32(g.min_x))) | (u > np.float64(np.float32(g.max_x))) |
                       (v < np.float64(np.float32(g.min_y))) | (v > np.float64(np.float32(g.max_y))))
            ok = front & inside
    if usable is not None:
        ok &= np.asarray(usable, bool)
    uv = np.where(ok[:, None], np.stack([u, v], 1).astype(np.float32), np.float32(0))
    return ok, uv.astype(np.float32), np.where(ok, xr, np.float32(0)).astype(np.float32)


def _log_ratio(ratio):
    """log of each positive finite float ratio through the C library; -inf / inf / nan as the C library gives them"""
    out = np.empty(ratio.shape, np.float64)
    for i, r in enumerate(ratio.astype(np.float64)):
        if r > 0 and math.isfinite(r):
            out[i] = math.log(r)
        elif r == 0:
            out[i] = -math.inf
        elif r == math.inf:
            out[i] = math.inf
        else:
            out[i] = math.nan
    return out


def predict_scale_level(dist_f, max_valid_dist, log_scale_factor, num_levels):
    """ceil(log_f(max_valid_dist / dist_f) / log_scale_factor) in float, clamped to [0, num_levels - 1] (NaN: 0)"""
    with np.errstate(all="ignore"):
        ratio = np.asarray(max_valid_dist, np.float32) / np.asarray(dist_f, np.float32)
        lg = _log_ratio(np.atleast_1d(ratio)).astype(np.float32)
        q = np.ceil(lg / np.float32(log_scale_factor))
        level = np.zeros(q.shape, np.int32)
        pos = q >= 0
        level[pos] = np.where(q[pos] >= np.float32(num_levels), num_levels - 1, np.minimum(q[pos], num_levels)).astype(np.int32)
    return level


def can_observe(g, pos_w, mean_normal, min_valid_dist, max_valid_dist, ray_cos_thr=0.5, usable=None):
    """-> observable (n,) bool, reproj_xy (n, 2) f32, x_right (n,) f32, pred_scale_level (n,) i32 (zeros where not observable)"""
    P = np.asarray(pos_w, np.float64).reshape(-1, 3)
    N = np.asarray(mean_normal, np.float64).reshape(-1, 3)
    lo_raw = np.asarray(min_valid_dist, np.float32); hi_raw = np.asarray(max_valid_dist, np.float32)
    ok, uv, xr = reproject(g, P, usable)
    C = np.array(g.cam_center[:], np.float64)
    with np.errstate(all="ignore"):
        v = P - C
        dist = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
        d = dist.astype(np.float32)
        lo = (0.7 * lo_raw.astype(np.float64)).astype(np.float32)
        hi = (1.3 * hi_raw.astype(np.float64)).astype(np.float32)
        ok &= (lo <= d) & (d <= hi)
        ray_cos = ((v[:, 0] * N[:, 0] + v[:, 1] * N[:, 1]) + v[:, 2] * N[:, 2]) / dist
        ok &= ~(ray_cos < np.float64(np.float32(ray_cos_thr)))
        level = predict_scale_level(d, hi_raw, g.log_scale_factor, g.num_scale_levels)
    level = np.where(ok, level, 0).astype(np.int32)
    uv = np.where(ok[:, None], uv, np.float32(0)).astype(np.float32)
    xr = np.where(ok, xr, np.float32(0)).astype(np.float32)
    return ok, uv, xr, level


def motion_direction(pose_cw_curr, pose_cw_last, is_monocular, true_baseline):
    if is_monocular:
        return False, False
    c = np.asarray(pose_cw_curr, np.float64).reshape(12)
    l = np.asarray(pose_cw_last, np.float64).reshape(12)
    wc = [-((c[i] * c[9] + c[3 + i] * c[10]) + c[6 + i] * c[11]) for i in range(3)]
    z = ((l[6] * wc[0] + l[7] * wc[1]) + l[8] * wc[2]) + l[11]
    return bool(z > true_baseline), bool(-z > true_baseline)
