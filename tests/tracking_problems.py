"""Seeded scenes and knife edges for the tracker's per-landmark geometry (frame::can_observe, the motion model's reprojection):
shared by the oracle test on the CPU and the device test."""
import math

import numpy as np

from openvslam_b200.match import frame_geometry
from openvslam_b200.optimize import camera

SCALE_FACTOR = 1.2
NUM_LEVELS = 8
LOG_SCALE_FACTOR = np.float32(math.log(SCALE_FACTOR))
SCALE_FACTORS = np.array([SCALE_FACTOR ** i for i in range(NUM_LEVELS)], np.float32)

# (model, camera kwargs, img_bounds): the fisheye and radial-division cameras reproject with the pinhole formula on undistorted
# keypoints, against bounds wider than the image
CAMERAS = {
    "mono": ("perspective", dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0), (0.0, 640.0, 0.0, 480.0)),
    "stereo": ("perspective", dict(fx=718.856, fy=718.856, cx=607.19, cy=185.21, focal_x_baseline=386.1448), (0.0, 1241.0, 0.0, 376.0)),
    "fisheye": ("fisheye", dict(fx=400.0, fy=400.0, cx=640.0, cy=480.0), (-212.4, 1492.4, -160.25, 1120.25)),
    "radial_division": ("radial_division", dict(fx=300.0, fy=300.0, cx=320.0, cy=240.0), (-35.5, 675.5, -20.75, 500.75)),
    "equirectangular": ("equirectangular", dict(cols=1920.0, rows=960.0), (0.0, 1920.0, 0.0, 960.0)),
}
SCENES = tuple(CAMERAS)


def rotation(rng, angle=0.3):
    w = rng.normal(size=3)
    w *= angle / np.linalg.norm(w)
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K


def pose12(R, t):
    return np.concatenate([np.asarray(R, np.float64).reshape(9), np.asarray(t, np.float64)])


def geometry(scene, pose_cw, log_scale_factor=LOG_SCALE_FACTOR, num_levels=NUM_LEVELS):
    model, kw, bounds = CAMERAS[scene]
    return frame_geometry(camera(model, **kw), bounds, pose_cw, num_levels, log_scale_factor)


def scene(name, n, seed, frac_behind=0.1):
    """A random pose and n landmarks around it: positions (a fraction behind the camera), mean normals near the viewing ray, and
    valid distances around the true distance (some outside the scale range) -> dict(geometry, pos_w, mean_normal, min_valid_dist,
    max_valid_dist, usable, pose_cw)."""
    rng = np.random.default_rng(seed)
    R = rotation(rng)
    t = rng.normal(size=3)
    pose = pose12(R, t)
    g = geometry(name, pose)
    center = -(R.T @ t)
    if name == "equirectangular":
        d = rng.normal(size=(n, 3))
    else:
        # directions in the camera frame, mostly inside a wide cone in front of it
        d = np.stack([rng.uniform(-0.9, 0.9, n), rng.uniform(-0.7, 0.7, n), np.ones(n)], 1)
        d[rng.random(n) < frac_behind, 2] *= -1
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    dist = rng.uniform(0.5, 30.0, n)
    pos_w = center + (d * dist[:, None]) @ R       # R^T applied to the camera-frame direction
    ray = (pos_w - center) / dist[:, None]
    nrm = ray + rng.normal(scale=0.6, size=(n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    # ratios max_valid / dist from 0.6 (outside the scale range) to 5 (beyond the last level)
    max_valid = (dist * np.exp(rng.uniform(math.log(0.6), math.log(5.0), n))).astype(np.float32)
    min_valid = (max_valid / np.float32(SCALE_FACTOR ** (NUM_LEVELS - 1)) * rng.uniform(0.5, 1.6, n)).astype(np.float32)
    usable = (rng.random(n) < 0.9).astype(np.uint8)
    return dict(geometry=g, pos_w=pos_w, mean_normal=nrm, min_valid_dist=min_valid, max_valid_dist=max_valid, usable=usable, pose_cw=pose)


def _f32_neighbours(v):
    v = np.float32(v)
    return [np.nextafter(v, np.float32(-np.inf)), v, np.nextafter(v, np.float32(np.inf))]


def knife_edges(equirectangular=False):
    """Landmarks at the conventions' edges, seen from the identity pose: z = 0 and -0.0; reprojections on each image bound and one
    ulp beyond; distances on each scaled bound and one float ulp either side; a ray cosine of exactly 0.5 and just below; a ratio
    below 1 and beyond the last level; quotients log_f(ratio) / log_scale_factor at an integer and one ulp of distance either
    side; NaN and +-inf positions.  The log scale factor is log_f(2), so that ratios 2 and 4 give the quotients 1 and 2 exactly.
    -> dict as scene() (geometry: fx = fy = 512, cx = 320, cy = 240, bounds 0 .. 640 x 0 .. 480, or a 1920 x 960 equirectangular)."""
    lsf = np.float32(math.log(2.0))
    if equirectangular:
        g = frame_geometry(camera("equirectangular", cols=1920.0, rows=960.0), (0.0, 1920.0, 0.0, 960.0), pose12(np.eye(3), np.zeros(3)),
                           NUM_LEVELS, lsf)
    else:
        g = frame_geometry(camera("perspective", fx=512.0, fy=512.0, cx=320.0, cy=240.0, focal_x_baseline=40.0), (0.0, 640.0, 0.0, 480.0),
                           pose12(np.eye(3), np.zeros(3)), NUM_LEVELS, lsf)
    P, N, lo, hi = [], [], [], []
    fwd = [0.0, 0.0, 1.0]

    def add(p, n=fwd, mn=0.1, mx=8.0):
        P.append(p); N.append(n); lo.append(mn); hi.append(mx)

    add([1.0, 1.0, 0.0]); add([1.0, 1.0, -0.0]); add([0.0, 0.0, -1.0])
    # the image bounds: u = 512 x + 320 on 0 and 640 at x = -+0.625, v = 512 y + 240 on 0 and 480 at y = -+0.46875 (z = 1)
    for x in (-0.625, 0.625):
        for e in _f32_neighbours(x):
            add([float(e), 0.0, 1.0], mn=0.1, mx=8.0)
        add([float(np.nextafter(x, -math.inf if x < 0 else math.inf)), 0.0, 1.0])
    for y in (-0.46875, 0.46875):
        add([0.0, y, 1.0])
        add([0.0, float(np.nextafter(y, -math.inf if y < 0 else math.inf)), 1.0])
    # the scaled distance bounds, with the landmark on the optical axis (dist = z exactly)
    for mn, mx in ((1.0, 8.0), (0.3, 3.7), (2.0, 2.1)):
        for b in (np.float32(0.7 * np.float32(mn)), np.float32(1.3 * np.float32(mx))):
            for z in _f32_neighbours(b):
                add([0.0, 0.0, float(z)], mn=mn, mx=mx)
    # the ray cosine: exactly 0.5, and the normal a little further off
    add([0.0, 0.0, 2.0], n=[math.sqrt(3.0) / 2.0, 0.0, 0.5])
    add([0.0, 0.0, 2.0], n=[math.sqrt(3.0) / 2.0, 0.0, float(np.nextafter(0.5, 0.0))])
    # ratio < 1 (level 0) and far beyond the last level (clamped)
    add([0.0, 0.0, 9.0], mn=0.1, mx=8.0)
    add([0.0, 0.0, 0.02], mn=0.01, mx=8.0)
    # quotients at the integers 1 and 2 (ratio 2 and 4 with max 8) and one float ulp of distance either side
    for z in (4.0, 2.0):
        for e in _f32_neighbours(z):
            add([0.0, 0.0, float(e)], mn=0.1, mx=8.0)
    # non-finite positions
    for p in ([math.nan, 0.0, 2.0], [0.0, math.nan, 2.0], [0.0, 0.0, math.nan], [math.inf, 0.0, 2.0], [-math.inf, 0.0, 2.0],
              [0.0, 0.0, math.inf], [0.0, 0.0, -math.inf], [0.0, math.inf, 2.0]):
        add(p)
    n = len(P)
    return dict(geometry=g, pos_w=np.array(P, np.float64), mean_normal=np.array(N, np.float64), min_valid_dist=np.array(lo, np.float32),
                max_valid_dist=np.array(hi, np.float32), usable=np.ones(n, np.uint8), pose_cw=pose12(np.eye(3), np.zeros(3)))
