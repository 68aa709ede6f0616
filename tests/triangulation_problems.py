"""Seeded scenes for the two-view triangulator and create_new_landmarks: keyframes observing one set of 3-D points, with
pixel noise, gross outliers, stereo keypoints, descriptors and BoW nodes shared between the views of a point, and landmark flags."""
import numpy as np

from openvslam_b200 import module, optimize

FX, FY, CX, CY, COLS, ROWS = 500.0, 500.0, 320.0, 240.0, 640, 480
EQ_COLS, EQ_ROWS = 2000.0, 1000.0
NUM_LEVELS = 8


def scale_tables():
    sf = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(NUM_LEVELS - 1, np.float32(1.2))]).astype(np.float32)).astype(np.float32)
    return sf, (sf * sf).astype(np.float32)


def rot(rng, deg):
    w = rng.normal(0, 1, 3); w *= np.deg2rad(deg) / np.linalg.norm(w)
    th = np.linalg.norm(w); k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def pose_of(R, c):
    """{R_cw, t_cw} of a camera with rotation R_cw and centre c"""
    return np.concatenate([R.reshape(9), -R @ c])


def bearing_equirect(x, y):
    lon = (x.astype(np.float64) / EQ_COLS - 0.5) * 2 * np.pi
    lat = -(y.astype(np.float64) / EQ_ROWS - 0.5) * np.pi
    return np.stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)], 1)


def make_scene(rng, n_points, model="perspective"):
    if model == "perspective":
        X = np.stack([rng.uniform(-8, 8, n_points), rng.uniform(-5, 5, n_points), rng.uniform(4, 30, n_points)], 1)
    else:
        d = rng.normal(0, 1, (n_points, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
        X = d * rng.uniform(3, 25, (n_points, 1))
    base = rng.integers(0, 256, (n_points, 32), dtype=np.uint8)
    return dict(X=X, base=base, angle=rng.uniform(0, 360, n_points), model=model)


def make_keyframe(rng, scene, centre, R, stereo_frac=0.0, n_nodes=40, noise_px=0.5, outlier_frac=0.05, has_lm_frac=0.2,
                  n_distractors=None, visible_frac=0.85, true_baseline=0.5, angle_offset=0.0, max_keypts=None):
    """A keyframe at `centre` with rotation R_cw observing part of the scene; returns (module.keyframe, point index of each
    keypoint or -1)."""
    X, model = scene["X"], scene["model"]
    pose = pose_of(R, centre)
    Xc = X @ R.T + pose[9:]
    sf, sig = scale_tables()
    if model == "perspective":
        cam = optimize.camera("perspective", FX, FY, CX, CY, focal_x_baseline=FX * true_baseline, cols=COLS, rows=ROWS)
        z = Xc[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = FX * Xc[:, 0] / z + CX; v = FY * Xc[:, 1] / z + CY
        vis = (z > 0.5) & (u >= 0) & (u < COLS) & (v >= 0) & (v < ROWS)
    else:
        cam = optimize.camera("equirectangular", cols=EQ_COLS, rows=EQ_ROWS)
        b = Xc / np.linalg.norm(Xc, axis=1, keepdims=True)
        u = EQ_COLS * (0.5 + np.arctan2(b[:, 0], b[:, 2]) / (2 * np.pi)); v = EQ_ROWS * (0.5 + np.arcsin(b[:, 1]) / np.pi)
        z = np.linalg.norm(Xc, axis=1)
        vis = np.ones(len(X), bool)
        stereo_frac = 0.0
    idx = np.flatnonzero(vis & (rng.random(len(X)) < visible_frac))
    if max_keypts is not None:
        idx = idx[:max_keypts]
    n = len(idx)
    nd = n // 4 if n_distractors is None else n_distractors
    octave = rng.integers(0, NUM_LEVELS, n + nd).astype(np.int32)
    s = sf[octave[:n]].astype(np.float64)
    noise = rng.normal(0, noise_px, (n, 2)) * s[:, None]
    out = rng.random(n) < outlier_frac
    noise[out] = rng.normal(0, 25.0, (out.sum(), 2))
    x = np.concatenate([u[idx] + noise[:, 0], rng.uniform(0, COLS if model == "perspective" else EQ_COLS, nd)]).astype(np.float32)
    y = np.concatenate([v[idx] + noise[:, 1], rng.uniform(0, ROWS if model == "perspective" else EQ_ROWS, nd)]).astype(np.float32)
    if model == "perspective":
        b = np.stack([(x.astype(np.float64) - CX) / FX, (y.astype(np.float64) - CY) / FY, np.ones(n + nd)], 1)
        b /= np.linalg.norm(b, axis=1, keepdims=True)
    else:
        b = bearing_equirect(x, y)
    # descriptors: the point's, a few bytes changed; distractors random
    desc = np.concatenate([scene["base"][idx], rng.integers(0, 256, (nd, 32), dtype=np.uint8)])
    for _ in range(2):
        byte = rng.integers(0, 32, n); desc[np.arange(n), byte] ^= (rng.integers(0, 256, n) & rng.integers(0, 256, n)).astype(np.uint8)
    node_pt = (scene["base"][:, 0].astype(np.int32) * 7 + scene["base"][:, 1]) % n_nodes
    node = np.concatenate([node_pt[idx], rng.integers(0, n_nodes, nd)]).astype(np.int32)
    node[rng.random(n + nd) < 0.02] = -1
    angle = np.concatenate([scene["angle"][idx] + angle_offset + rng.normal(0, 2.0, n), rng.uniform(0, 360, nd)]) % 360
    has_lm = (rng.random(n + nd) < has_lm_frac).astype(np.uint8)
    xr = dp = None
    if stereo_frac > 0:
        st = rng.random(n + nd) < stereo_frac
        depth = np.concatenate([z[idx], rng.uniform(4, 30, nd)]) * (1 + rng.normal(0, 0.002, n + nd))
        dp = np.where(st, depth, -1.0).astype(np.float32)
        xr = np.where(st, x - FX * true_baseline / np.where(st, depth, 1.0) + rng.normal(0, 0.3, n + nd), -1.0).astype(np.float32)
        # a right-image x is never negative in the reference's stereo matcher
        bad = st & (xr < 0)
        xr[bad] = -1.0; dp[bad] = -1.0
    perm = rng.permutation(n + nd)                # keypoints are not stored in point order
    kf = module.keyframe(pose, cam, 1.2, sf, sig, x[perm], y[perm], octave[perm], b[perm], angle=angle[perm].astype(np.float32),
                         stereo_x_right=None if xr is None else xr[perm], depths=None if dp is None else dp[perm],
                         true_baseline=true_baseline, descriptors=desc[perm], has_landmark=has_lm[perm], bow_node=node[perm])
    pt = np.concatenate([idx, -np.ones(nd, np.int64)])[perm]
    return kf, pt


def e12_epipole(kf1, kf2):
    """E_12 (b1' E_12 b2 = 0) and the bearing of camera centre 1 seen from keyframe 2, from the poses, as the reference forms them"""
    R1, t1 = kf1.pose_cw[:9].reshape(3, 3), kf1.pose_cw[9:]
    R2, t2 = kf2.pose_cw[:9].reshape(3, 3), kf2.pose_cw[9:]
    R12 = R1 @ R2.T
    t12 = -R12 @ t2 + t1
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    c1 = -R1.T @ t1
    e = R2 @ c1 + t2
    return tx @ R12, e / np.linalg.norm(e)


def neighbourhood(seed, n1, B, model="perspective", stereo_frac=0.0, n_nodes=40, spacing=0.4):
    """Keyframe 1 and B neighbours around it (some close, some far); -> kf1, [kf2], E_12 (B, 3, 3), epipoles (B, 3)"""
    rng = np.random.default_rng(seed)
    scene = make_scene(rng, int(n1 * 1.4), model)
    kf1, _ = make_keyframe(rng, scene, np.zeros(3), rot(rng, 1.0), stereo_frac, n_nodes, max_keypts=int(n1 * 0.8),
                           n_distractors=n1 - int(n1 * 0.8))
    kf1 = _trim(kf1, n1)
    nbs, Es, eps = [], [], []
    for b in range(B):
        c = np.array([spacing * (b + 1) * (-1) ** b, rng.normal(0, 0.05), rng.normal(0, 0.1)])
        if b % 5 == 4:
            c *= 0.05                                # nearly the same place: stereo parallax wins
        kf2, _ = make_keyframe(rng, scene, c, rot(rng, 3.0), stereo_frac, n_nodes, angle_offset=rng.uniform(-20, 20))
        E, e = e12_epipole(kf1, kf2)
        nbs.append(kf2); Es.append(E); eps.append(e)
    return kf1, nbs, np.array(Es).reshape(B, 3, 3), np.array(eps).reshape(B, 3)


def _trim(kf, n):
    """the first n keypoints of a keyframe (every per-keypoint array cut the same way)"""
    sl = slice(0, min(n, kf.num_keypts))
    return module.keyframe(kf.pose_cw, kf.camera, kf.scale_factor, kf.scale_factors, kf.level_sigma_sq, kf.keypts["x"][sl], kf.keypts["y"][sl],
                           kf.keypts["octave"][sl], kf.bearings[sl], angle=kf.keypts["angle"][sl],
                           stereo_x_right=None if kf.stereo_x_right is None else kf.stereo_x_right[sl],
                           depths=None if kf.depths is None else kf.depths[sl], true_baseline=kf.true_baseline,
                           descriptors=kf.descriptors[sl], has_landmark=kf.has_landmark[sl], bow_node=kf.bow_node[sl])


def pair_problem(seed, m, model="perspective", stereo_frac=0.0, spacing=0.4):
    """Two keyframes and m keypoint pairs: mostly true correspondences, the rest random pairs."""
    rng = np.random.default_rng(seed)
    scene = make_scene(rng, max(2 * m, 64), model)
    kf1, p1 = make_keyframe(rng, scene, np.zeros(3), rot(rng, 1.0), stereo_frac)
    c = np.array([spacing, rng.normal(0, 0.05), rng.normal(0, 0.1)])
    kf2, p2 = make_keyframe(rng, scene, c, rot(rng, 3.0), stereo_frac)
    inv2 = {int(p): i for i, p in enumerate(p2) if p >= 0}
    true = [(i, inv2[int(p)]) for i, p in enumerate(p1) if p >= 0 and int(p) in inv2]
    true = np.array(true, np.int32).reshape(-1, 2)
    k = min(len(true), int(0.7 * m))
    sel = true[rng.permutation(len(true))[:k]]
    rnd = np.stack([rng.integers(0, kf1.num_keypts, m - k), rng.integers(0, kf2.num_keypts, m - k)], 1).astype(np.int32)
    pairs = np.concatenate([sel, rnd])[rng.permutation(m)] if m else np.zeros((0, 2), np.int32)
    return kf1, kf2, pairs.astype(np.int32)
