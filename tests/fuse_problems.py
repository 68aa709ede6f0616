"""Seeded scenes and knife edges for match::fuse::replace_duplication (the geometry of fuse_observe and the batched search over
target keyframes): shared by the oracle test on the CPU and the device test."""
import math

import numpy as np

from openvslam_b200.match import camera_grid, frame_geometry, fuse_target
from openvslam_b200.optimize import camera
import tracking_problems as TP

NUM_LEVELS = TP.NUM_LEVELS
SCALE_FACTORS = TP.SCALE_FACTORS
INV_LEVEL_SIGMA_SQ = (1.0 / (SCALE_FACTORS.astype(np.float64) ** 2)).astype(np.float32)

# (model, camera kwargs, img_bounds, stereo)
CAMERAS = {
    "mono": ("perspective", dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0), (0.0, 640.0, 0.0, 480.0), False),
    "stereo": ("perspective", dict(fx=718.856, fy=718.856, cx=607.19, cy=185.21, focal_x_baseline=386.1448), (0.0, 1241.0, 0.0, 376.0), True),
    "equirectangular": ("equirectangular", dict(cols=1920.0, rows=960.0), (0.0, 1920.0, 0.0, 960.0), False),
}


def _project(model, kw, pose, P):
    R, t = pose[:9].reshape(3, 3), pose[9:]
    pc = P @ R.T + t
    if model == "equirectangular":
        b = pc / np.linalg.norm(pc, axis=1, keepdims=True)
        u = kw["cols"] * (0.5 + np.arctan2(b[:, 0], b[:, 2]) / (2 * math.pi))
        v = kw["rows"] * (0.5 + np.arcsin(b[:, 1]) / math.pi)
        return u, v, pc[:, 2], np.ones(len(P), bool)
    with np.errstate(all="ignore"):
        u = kw["fx"] * pc[:, 0] / pc[:, 2] + kw["cx"]
        v = kw["fy"] * pc[:, 1] / pc[:, 2] + kw["cy"]
    return u, v, pc[:, 2], pc[:, 2] > 0


def landmarks(nlm, rng, equirectangular=False):
    """nlm landmarks in front of the origin (all around it for equirectangular): pos_w, mean normals near the ray from the origin,
    raw valid distances around the distance (some outside the range), descriptors."""
    if equirectangular:
        d = rng.normal(size=(nlm, 3))
    else:
        d = np.stack([rng.uniform(-0.6, 0.6, nlm), rng.uniform(-0.45, 0.45, nlm), np.ones(nlm)], 1)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    dist = rng.uniform(2.0, 20.0, nlm)
    pos = d * dist[:, None]
    nrm = d + rng.normal(scale=0.4, size=(nlm, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    max_valid = (dist * np.exp(rng.uniform(math.log(0.7), math.log(4.0), nlm))).astype(np.float32)
    min_valid = (max_valid / np.float32(TP.SCALE_FACTOR ** (NUM_LEVELS - 1)) * rng.uniform(0.5, 1.5, nlm)).astype(np.float32)
    desc = rng.integers(0, 256, size=(nlm, 32), dtype=np.uint8)
    return dict(pos_w=pos, mean_normal=nrm, min_valid_dist=min_valid, max_valid_dist=max_valid, lm_desc=desc)


def _flip(desc, nbits, rng):
    out = desc.copy()
    for i in range(len(out)):
        for b in rng.choice(256, int(nbits[i]), replace=False):
            out[i, b // 8] ^= np.uint8(1 << (b % 8))
    return out


def target(scene, lms, nkp, rng, pose=None):
    """A target keyframe near the origin whose keypoints sit near the reprojections of most landmarks it sees (jittered, at about
    the predicted level, a few descriptor bits flipped, some far off), plus clutter; nkp keypoints at most.  -> (fuse_target,
    dict of its arrays for the oracle)."""
    model, kw, bounds, stereo = CAMERAS[scene]
    if pose is None:
        pose = TP.pose12(TP.rotation(rng, 0.05), rng.normal(scale=0.2, size=3))
    g = frame_geometry(camera(model, **kw), bounds, pose, NUM_LEVELS, TP.LOG_SCALE_FACTOR)
    grid = camera_grid(*bounds)
    P = lms["pos_w"]
    u, v, z, front = _project(model, kw, np.asarray(pose, np.float64), P)
    inside = front & (u >= bounds[0]) & (u < bounds[1]) & (v >= bounds[2]) & (v < bounds[3])
    seen = np.flatnonzero(inside & (rng.random(len(P)) < 0.7))[: (nkp * 3) // 4]
    ns = len(seen)
    dist = np.linalg.norm(P[seen] - np.asarray(g.cam_center[:]), axis=1)
    lvl = np.clip(np.ceil(np.log(lms["max_valid_dist"][seen] / dist) / math.log(TP.SCALE_FACTOR)), 0, NUM_LEVELS - 1).astype(np.int32)
    lvl = np.clip(lvl - rng.integers(0, 2, ns), 0, NUM_LEVELS - 1)
    x = (u[seen] + rng.normal(scale=0.8, size=ns) * SCALE_FACTORS[lvl]).astype(np.float32)
    y = (v[seen] + rng.normal(scale=0.8, size=ns) * SCALE_FACTORS[lvl]).astype(np.float32)
    desc = _flip(lms["lm_desc"][seen], np.where(rng.random(ns) < 0.85, rng.integers(0, 30, ns), rng.integers(40, 90, ns)), rng)
    nc = max(nkp - ns, 0)
    cx = rng.uniform(bounds[0], bounds[1], nc).astype(np.float32); cy = rng.uniform(bounds[2], bounds[3], nc).astype(np.float32)
    x = np.concatenate([x, cx]); y = np.concatenate([y, cy])
    octave = np.concatenate([lvl, rng.integers(0, NUM_LEVELS, nc)]).astype(np.int32)
    desc = np.concatenate([desc, rng.integers(0, 256, size=(nc, 32), dtype=np.uint8)])
    perm = rng.permutation(len(x))
    x, y, octave, desc = x[perm], y[perm], octave[perm], desc[perm]
    xr = None
    if stereo:
        zz = np.concatenate([z[seen], rng.uniform(2.0, 20.0, nc)])[perm]
        xr = np.where(rng.random(len(x)) < 0.7, x - np.float32(kw["focal_x_baseline"]) / zz + rng.normal(scale=0.5, size=len(x)), -1.0).astype(np.float32)
    arrays = dict(geometry=g, x=x, y=y, octave=octave, desc=desc, x_right=xr, grid=grid)
    return fuse_target(g, SCALE_FACTORS, INV_LEVEL_SIGMA_SQ, x, y, octave, desc, grid, x_right=xr), arrays


def batch(scene, B, nlm, nkp, q_per_target, seed, skip_frac=0.0, empty=()):
    """B targets over one landmark table; target t gets q_per_target[t] queries drawn from the landmarks (-1 for a fraction
    skip_frac); the targets listed in `empty` have no keypoints.  -> (targets, arrays, lms, q_off, q_lm)"""
    rng = np.random.default_rng(seed)
    lms = landmarks(nlm, rng, scene == "equirectangular")
    targets, arrays = [], []
    for t in range(B):
        ft, a = target(scene, lms, 0 if t in empty else nkp, rng)
        targets.append(ft); arrays.append(a)
    q_off = np.concatenate([[0], np.cumsum(q_per_target)]).astype(np.int32)
    Q = int(q_off[-1])
    q_lm = rng.integers(0, nlm, Q).astype(np.int32) if nlm else np.full(Q, -1, np.int32)
    if skip_frac:
        q_lm[rng.random(Q) < skip_frac] = -1
    return targets, arrays, lms, q_off, q_lm


def _f64_neighbours(v):
    v = float(v)
    return [np.nextafter(v, -math.inf), v, np.nextafter(v, math.inf)]


def knife_edges(equirectangular=False):
    """The tracker's knife edges (tracking_problems.knife_edges: z = +-0, the image bounds, the quotients at an integer, NaN and
    +-inf positions, the ray at exactly 0.5) plus the fuse gates' own: distances exactly on (double)(float)(0.7 min) and
    (double)(float)(1.3 max) and one double ulp either side, v . n == 0.5 dist exactly and one ulp of the normal below."""
    s = TP.knife_edges(equirectangular)
    P, N, lo, hi = [list(s["pos_w"])], [list(s["mean_normal"])], [list(s["min_valid_dist"])], [list(s["max_valid_dist"])]
    extra = []
    for mn, mx in ((1.0, 8.0), (0.3, 3.7), (2.0, 2.1), (0.11, 5.3)):
        for b in (np.float32(0.7 * np.float64(np.float32(mn))), np.float32(1.3 * np.float64(np.float32(mx)))):
            for z in _f64_neighbours(np.float64(b)):
                extra.append(([0.0, 0.0, z], [0.0, 0.0, 1.0], mn, mx))
    # v . n = 0.5 dist: the normal at 60 degrees from the axis, dist = 2 and 3
    for z in (2.0, 3.0):
        extra.append(([0.0, 0.0, z], [math.sqrt(3.0) / 2.0, 0.0, 0.5], 0.1, 8.0))
        extra.append(([0.0, 0.0, z], [math.sqrt(3.0) / 2.0, 0.0, float(np.nextafter(0.5, 0.0))], 0.1, 8.0))
    P.append([e[0] for e in extra]); N.append([e[1] for e in extra]); lo.append([e[2] for e in extra]); hi.append([e[3] for e in extra])
    out = dict(s)
    out["pos_w"] = np.concatenate([np.asarray(p, np.float64).reshape(-1, 3) for p in P])
    out["mean_normal"] = np.concatenate([np.asarray(p, np.float64).reshape(-1, 3) for p in N])
    out["min_valid_dist"] = np.concatenate([np.asarray(p, np.float32) for p in lo])
    out["max_valid_dist"] = np.concatenate([np.asarray(p, np.float32) for p in hi])
    out["usable"] = np.ones(len(out["pos_w"]), np.uint8)
    return out
