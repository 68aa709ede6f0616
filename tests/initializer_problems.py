"""Two-view map-initialisation problems (initialize::perspective, initialize::bearing_vector) and an independent numpy restatement of
what happens after the solvers: the decompositions on numpy's SVD (with the library's column sign rule), a vectorised check_pose
(np.sort for the k-th smallest cos_parallax) and find_most_plausible_pose.  Extends tests/two_view_problems.py: view 1 is the
reference (the origin), p_cur = R p_ref + t; the perspective camera is K = [[500, 0, 320], [0, 500, 240], [0, 0, 1]] (640 x 480),
the equirectangular one 1920 x 960."""
import numpy as np
from scipy.spatial.transform import Rotation

from two_view_problems import K, KI, _project

PERSPECTIVE = dict(model=0, fx=500.0, fy=500.0, cx=320.0, cy=240.0, cols=640.0, rows=480.0)
EQUIRECT = dict(model=1, fx=0.0, fy=0.0, cx=0.0, cy=0.0, cols=1920.0, rows=960.0)
SMALL_COS = 0.99998


def perspective_bearings(kp):
    r = np.concatenate([np.asarray(kp, np.float64), np.ones((len(kp), 1))], 1) @ KI.T
    return r / np.linalg.norm(r, axis=1, keepdims=True)


def equirect_project(p, cam=EQUIRECT):
    b = p / np.linalg.norm(p, axis=1, keepdims=True)
    lat, lon = -np.arcsin(b[:, 1]), np.arctan2(b[:, 0], b[:, 2])
    return np.stack([cam["cols"] * (0.5 + lon / (2 * np.pi)), cam["rows"] * (0.5 - lat / np.pi)], 1)


def equirect_bearings(kp, cam=EQUIRECT):
    kp = np.asarray(kp, np.float64)
    lon = (kp[:, 0] / cam["cols"] - 0.5) * 2 * np.pi
    lat = -(kp[:, 1] / cam["rows"] - 0.5) * np.pi
    return np.stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)], 1)


def problem(m, scene="general", wrong=0.0, noise=0.0, seed=0, baseline=0.4, camera="perspective", extra=None):
    """m matches among m + 20 % + 5 keypoints per view (the rest unmatched), as a dict with cam, keypts / bearings per view,
    ref_matches_with_cur, the truth R, t, nrm (the plane's normal for "planar"), p_ref (m, 3) and the matched reference indices.
    scene: "general" (depths 4..10 m), "planar" (a tilted plane 6 m away), "rotation" (t = 0); baseline scales t; `wrong` of the
    matches take another match's current keypoint; noise is the pixel noise on both views; extra: the unmatched keypoints of the
    reference view (the current view then has 3 more)."""
    rng = np.random.default_rng(seed)
    n1 = n2 = m + m // 5 + 5
    if extra is not None:
        n1, n2 = m + extra, m + extra + 3
    R = Rotation.from_rotvec(rng.normal(size=3) * 0.08).as_matrix()
    t = np.zeros(3) if scene == "rotation" else rng.normal(size=3) * baseline
    nrm = np.array([rng.normal() * 0.3, rng.normal() * 0.3, 1.0])
    nrm /= np.linalg.norm(nrm)
    if camera == "perspective":
        cam = PERSPECTIVE
        uv = np.stack([rng.uniform(20.0, 620.0, m), rng.uniform(20.0, 460.0, m)], 1)
        ray = np.concatenate([uv, np.ones((m, 1))], 1) @ KI.T
    else:
        cam = EQUIRECT
        ray = rng.normal(size=(m, 3))
        ray /= np.linalg.norm(ray, axis=1, keepdims=True)
    z = 6.0 / (ray @ nrm) if scene == "planar" else rng.uniform(4.0, 10.0, m)
    p1 = ray * z[:, None]
    p2 = p1 @ R.T + t
    proj = _project if camera == "perspective" else equirect_project
    x1, x2 = proj(p1), proj(p2)
    if noise > 0.0:
        x1 = x1 + rng.normal(size=x1.shape) * noise
        x2 = x2 + rng.normal(size=x2.shape) * noise
    w, h = cam["cols"], cam["rows"]
    k1 = np.stack([rng.uniform(0.0, w, n1), rng.uniform(0.0, h, n1)], 1)
    k2 = np.stack([rng.uniform(0.0, w, n2), rng.uniform(0.0, h, n2)], 1)
    s1, s2 = rng.permutation(n1)[:m], rng.permutation(n2)[:m]
    k1[s1] = x1
    k2[s2] = x2
    s2w = s2.copy()
    nb = int(round(wrong * m))
    if nb and m > 1:
        sel = rng.choice(m, nb, replace=False)
        s2w[sel] = s2[(sel + 1 + rng.integers(0, m - 1, nb)) % m]
    k1 = np.ascontiguousarray(k1, np.float32); k2 = np.ascontiguousarray(k2, np.float32)
    bear = perspective_bearings if camera == "perspective" else equirect_bearings
    rm = -np.ones(n1, np.int32)
    rm[s1] = s2w
    return dict(cam=cam, keypts_ref=k1, keypts_cur=k2, bearings_ref=bear(k1), bearings_cur=bear(k2), ref_matches_with_cur=rm,
                R=R, t=t, nrm=nrm, p_ref=p1, matched_ref=s1, perspective=camera == "perspective")


def oracle_args(p):
    return (p["perspective"], p["cam"], p["cam"], p["keypts_ref"], p["bearings_ref"], p["keypts_cur"], p["bearings_cur"],
            p["ref_matches_with_cur"])


# ------------------------------------------------------------------ numpy restatement
def canonical_columns(V):
    """each column signed so that its largest-magnitude entry (first on ties) is positive"""
    V = V.copy()
    for k in range(3):
        if V[np.argmax(np.abs(V[:, k])), k] < 0:
            V[:, k] = -V[:, k]
    return V


def svd3(A, third_by_cross=False):
    """numpy's SVD with the library's sign rule: V canonical, u_i = A v_i / d_i (u_3 = u_1 x u_2 with third_by_cross)"""
    _, d, Vt = np.linalg.svd(A)
    V = canonical_columns(Vt.T)
    U = np.zeros((3, 3))
    for k in range(2 if third_by_cross else 3):
        U[:, k] = A @ V[:, k] / d[k]
    if third_by_cross:
        U[:, 2] = np.cross(U[:, 0], U[:, 1])
    return U, d, V


def decompose_homography(H, cam_1, cam_2):
    Kf = lambda c: np.array([[c["fx"], 0, c["cx"]], [0, c["fy"], c["cy"]], [0, 0, 1.0]])
    A = np.linalg.inv(Kf(cam_2)) @ H @ Kf(cam_1)
    U, d, V = svd3(A)
    d1, d2, d3 = d
    if d1 / d2 < 1.00001 or d2 / d3 < 1.00001:
        return None
    s = np.linalg.det(U) * np.linalg.det(V)
    a1 = np.sqrt((d1 ** 2 - d2 ** 2) / (d1 ** 2 - d3 ** 2)); a3 = np.sqrt((d2 ** 2 - d3 ** 2) / (d1 ** 2 - d3 ** 2))
    x1 = [a1, a1, -a1, -a1]; x3 = [a3, -a3, a3, -a3]
    root = np.sqrt((d1 ** 2 - d2 ** 2) * (d2 ** 2 - d3 ** 2))
    Rs, ts, ns = [], [], []
    for neg in (0, 1):
        den = (d1 - d3) * d2 if neg else (d1 + d3) * d2
        sn = root / den
        c = (d1 * d3 - d2 ** 2) / den if neg else (d2 ** 2 + d1 * d3) / den
        for i, si in enumerate([sn, -sn, -sn, sn]):
            Rp = np.array([[c, 0, si], [0, -1, 0], [si, 0, -c]]) if neg else np.array([[c, 0, -si], [0, 1, 0], [si, 0, c]])
            Rs.append(s * U @ Rp @ V.T)
            tt = U @ (np.array([x1[i], 0, x3[i] if neg else -x3[i]]) * ((d1 + d3) if neg else (d1 - d3)))
            ts.append(tt / np.linalg.norm(tt))
            n = V @ np.array([x1[i], 0, x3[i]])
            ns.append(-n if n[2] < 0 else n)
    return np.array(Rs), np.array(ts), np.array(ns)


def decompose_essential(E):
    U, d, V = svd3(E, True)
    t = U[:, 2] / np.linalg.norm(U[:, 2])
    W = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]])
    Rs = []
    for M in (U @ W @ V.T, U @ W.T @ V.T):
        Rs.append(-M if np.linalg.det(M) < 0 else M)
    return np.array([Rs[0], Rs[0], Rs[1], Rs[1]]), np.array([t, -t, t, -t])


def decompose_fundamental(F, cam_1, cam_2):
    Kf = lambda c: np.array([[c["fx"], 0, c["cx"]], [0, c["fy"], c["cy"]], [0, 0, 1.0]])
    return decompose_essential(Kf(cam_2).T @ F @ Kf(cam_1))


def triangulate(b1, b2, R, t):
    """the reference's linear triangulation per match (numpy's SVD on the 4 x 4 A), vectorised"""
    P1 = np.hstack([np.eye(3), np.zeros((3, 1))]); P2 = np.hstack([R, t[:, None]])
    A = np.stack([b1[:, :1] * P1[2] - b1[:, 2:3] * P1[0], b1[:, 1:2] * P1[2] - b1[:, 2:3] * P1[1],
                  b2[:, :1] * P2[2] - b2[:, 2:3] * P2[0], b2[:, 1:2] * P2[2] - b2[:, 2:3] * P2[1]], 1)
    v = np.linalg.svd(A)[2][:, -1]
    with np.errstate(divide="ignore", invalid="ignore"):
        return v[:, :3] / v[:, 3:4]


def reproject(cam, p):
    if cam["model"] == 1:
        return np.ones(len(p), bool), equirect_project(p, cam)
    z = p[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = np.stack([cam["fx"] * p[:, 0] / z + cam["cx"], cam["fy"] * p[:, 1] / z + cam["cy"]], 1)
    return z > 0, uv


def check_pose(R, t, cam_ref, cam_cur, b_ref, b_cur, kp_ref, kp_cur, inlier, thr_sq=4.0, depth_is_positive=True):
    """-> (valid (m,), small (m,), p (m, 3), cos (m,) float32, margins: the smallest distance of each match to the thresholds it
    was decided by, for the comparison with the oracle)"""
    p = triangulate(b_ref, b_cur, R, t)
    c = -R.T @ t
    q = p - c
    with np.errstate(invalid="ignore", divide="ignore"):
        cos = ((p * q).sum(1) / (np.linalg.norm(p, axis=1) * np.linalg.norm(q, axis=1))).astype(np.float32)
    finite = np.isfinite(p).all(1) & ~np.isnan(cos)
    small = SMALL_COS < cos
    ok = inlier & finite
    if depth_is_positive:
        z2 = (p @ R.T + t)[:, 2]
        ok &= small | ((p[:, 2] > 0) & (z2 > 0))
    v1, uv1 = reproject(cam_ref, p)
    v2, uv2 = reproject(cam_cur, p @ R.T + t)
    e1 = ((uv1 - kp_ref) ** 2).sum(1); e2 = ((uv2 - kp_cur) ** 2).sum(1)
    ok &= v1 & v2 & ~(thr_sq < e1) & ~(thr_sq < e2)
    margin = np.minimum(np.abs(e1 - thr_sq) / thr_sq, np.abs(e2 - thr_sq) / thr_sq)
    margin = np.minimum(margin, np.abs(cos.astype(np.float64) - SMALL_COS))
    if depth_is_positive:
        margin = np.minimum(margin, np.minimum(np.abs(p[:, 2]), np.abs(z2)) / np.linalg.norm(p, axis=1))
    return ok, small, p, cos, margin


def kth_cos(cos_valid):
    if len(cos_valid) == 0:
        return np.float32(1.0)
    return np.sort(cos_valid)[min(50, len(cos_valid) - 1)]


def choose(counts, coss, min_num=50, parallax_deg=1.0):
    best = int(np.argmax(counts))
    if counts[best] < min_num:
        return 3, best
    if (0.8 * counts[best] < np.asarray(counts)).sum() > 1:
        return 4, best
    if np.cos(np.radians(parallax_deg)) < float(coss[best]):
        return 5, best
    return 0, best
