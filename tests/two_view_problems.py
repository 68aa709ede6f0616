"""Two-view keypoint problems for the homography and fundamental-matrix RANSAC solvers (solve::homography_solver,
solve::fundamental_solver: perspective map initialisation) and an independent numpy restatement of their arithmetic: the
normalisation in float32, the DLT and the eight-point algorithm with numpy's SVD on A (not the Jacobi on A^T A) and an SVD rank-2
projection, and a vectorised check_inliers.  View 1 is the origin; p_2 = R p_1 + t; K = [[500, 0, 320], [0, 500, 240], [0, 0, 1]]
(640 x 480).  H_21 maps pixels of view 1 to view 2 (p2 ~ H_21 p1), F_21 satisfies p2^T F_21 p1 = 0."""
import numpy as np
from scipy.spatial.transform import Rotation

from pnp_problems import sample as _sample

MIN_SET = 8
SCORE_THR = float(np.float32(5.991))
CHI_F = float(np.float32(3.841))
K = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
KI = np.linalg.inv(K)


def sample(seed, k, n):
    return _sample(seed, k, n, MIN_SET)


def skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _project(p):
    q = p @ K.T
    return q[:, :2] / q[:, 2:3]


def problem(m, scene="general", wrong=0.25, noise=0.0, seed=0, n1=None, n2=None):
    """m matches between view 1 and view 2, among n1 / n2 keypoints (default m + 20 % + 5: the extra keypoints are uniform in
    the image and unmatched, so that normalising over all keypoints differs from normalising over the matched ones).  scene:
    "general" (depths 4..10 m), "planar" (one plane about 6 m away, tilted) or "rotation" (t = 0).  `wrong` of the matches get the
    view-2 keypoint of another match; `noise` is the standard deviation of the pixel noise on both views."""
    rng = np.random.default_rng(seed)
    n1 = m + m // 5 + 5 if n1 is None else n1
    n2 = m + m // 5 + 5 if n2 is None else n2
    R = Rotation.from_rotvec(rng.normal(size=3) * 0.08).as_matrix()
    t = np.zeros(3) if scene == "rotation" else rng.normal(size=3) * 0.4
    uv = np.stack([rng.uniform(20.0, 620.0, m), rng.uniform(20.0, 460.0, m)], 1)
    ray = np.concatenate([uv, np.ones((m, 1))], 1) @ KI.T
    nrm = np.array([rng.normal() * 0.3, rng.normal() * 0.3, 1.0])
    nrm /= np.linalg.norm(nrm)
    d = 6.0
    if scene == "planar":
        z = d / (ray @ nrm)
    else:
        z = rng.uniform(4.0, 10.0, m)
    p1 = ray * z[:, None]
    p2 = p1 @ R.T + t
    x1, x2 = _project(p1), _project(p2)
    if noise > 0.0:
        x1 = x1 + rng.normal(size=x1.shape) * noise
        x2 = x2 + rng.normal(size=x2.shape) * noise
    k1 = np.stack([rng.uniform(0.0, 640.0, n1), rng.uniform(0.0, 480.0, n1)], 1)
    k2 = np.stack([rng.uniform(0.0, 640.0, n2), rng.uniform(0.0, 480.0, n2)], 1)
    s1, s2 = rng.permutation(n1)[:m], rng.permutation(n2)[:m]
    k1[s1] = x1
    k2[s2] = x2
    matches = np.stack([s1, s2], 1)
    bad = np.zeros(m, bool)
    nb = int(round(wrong * m))
    if nb and m > 1:
        sel = rng.choice(m, nb, replace=False)
        other = (sel + 1 + rng.integers(0, m - 1, nb)) % m
        matches[sel, 1] = s2[other]
        bad[sel] = True
    H_true = K @ (R + np.outer(t, nrm) / d) @ KI
    F_true = KI.T @ skew(t) @ R @ KI
    return dict(keypts_1=np.ascontiguousarray(k1, np.float32), keypts_2=np.ascontiguousarray(k2, np.float32),
                matches_12=np.ascontiguousarray(matches, np.int32), bad=bad, R=R, t=t, H_true=H_true, F_true=F_true, scene=scene)


def degenerate(kind, m=40, seed=0):
    """coincident (every match the same pair of keypoints), collinear (matched keypoints on one image line in both views), planar
    (for F) or rotation"""
    if kind in ("planar", "rotation"):
        return problem(m, scene=kind, wrong=0.0, seed=seed)
    p = problem(m, wrong=0.0, seed=seed)
    k1, k2, mt = p["keypts_1"].copy(), p["keypts_2"].copy(), p["matches_12"]
    if kind == "coincident":
        k1[mt[:, 0]] = k1[mt[0, 0]]
        k2[mt[:, 1]] = k2[mt[0, 1]]
    else:
        s = np.linspace(0.0, 1.0, m, dtype=np.float32)
        k1[mt[:, 0]] = np.stack([100 + 400 * s, 50 + 300 * s], 1)
        k2[mt[:, 1]] = np.stack([120 + 380 * s, 60 + 280 * s], 1)
    return dict(p, keypts_1=np.ascontiguousarray(k1), keypts_2=np.ascontiguousarray(k2))


def gpu_problem(p):
    return dict(keypts_1=p["keypts_1"], keypts_2=p["keypts_2"], matches_12=p["matches_12"])


# ------------------------------------------------------------------ numpy restatement
def normalize(xy):
    """float32 throughout; np.cumsum is the sequential running sum (np.sum is pairwise) -> (normalised, (mx, my, ix, iy))"""
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    n = np.float32(len(xy))
    mean = np.array([np.cumsum(xy[:, a], dtype=np.float32)[-1] / n for a in (0, 1)], np.float32)
    c = (xy - mean).astype(np.float32)
    dev = np.array([np.cumsum(np.abs(c[:, a]), dtype=np.float32)[-1] / n for a in (0, 1)], np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.array([np.float32(1.0 / np.float64(dev[a])) for a in (0, 1)], np.float32)
        return (c * inv).astype(np.float32), np.array([mean[0], mean[1], inv[0], inv[1]], np.float32)


def T_of(T4):
    mx, my, ix, iy = (np.float32(v) for v in T4)
    return np.array([[float(ix), 0.0, float(-mx * ix)], [0.0, float(iy), float(-my * iy)], [0.0, 0.0, 1.0]])


def T2inv_of(T4):
    mx, my, ix, iy = (float(v) for v in T4)
    return np.array([[1.0 / ix, 0.0, mx], [0.0, 1.0 / iy, my], [0.0, 0.0, 1.0]])


def canonical(M):
    f = M.ravel()
    return M * (-1.0 if f[np.argmax(np.abs(f))] < 0 else 1.0)


def design(model, q1, q2):
    """A of the normalised points (float32 -> float64): 2 rows per match for H, 1 for F"""
    x1, y1 = q1[:, 0].astype(np.float64), q1[:, 1].astype(np.float64)
    x2, y2 = q2[:, 0].astype(np.float64), q2[:, 1].astype(np.float64)
    o, z = np.ones_like(x1), np.zeros_like(x1)
    if model == "H":
        r0 = np.stack([z, z, z, -x1, -y1, -o, y2 * x1, y2 * y1, y2], 1)
        r1 = np.stack([x1, y1, o, z, z, z, -x2 * x1, -x2 * y1, -x2], 1)
        return np.stack([r0, r1], 1).reshape(-1, 9)
    return np.stack([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, o], 1)


def solve_normalised(model, q1, q2):
    """the model in normalised coordinates, canonical sign: the right singular vector of A's smallest singular value; for F then
    the SVD rank-2 projection"""
    M = np.linalg.svd(design(model, q1, q2))[2][-1].reshape(3, 3)
    if model == "F":
        U, S, Vt = np.linalg.svd(M)
        M = U @ np.diag([S[0], S[1], 0.0]) @ Vt
    return canonical(M)


def denormalise(model, Mn, T4_1, T4_2):
    L = T2inv_of(T4_2) if model == "H" else T_of(T4_2).T
    return canonical(L @ Mn @ T_of(T4_1))


def chis(model, M, k1, k2, matches, sigma=1.0):
    """(chi1, chi2) per match in the solver's order"""
    iss = float(np.float32(1.0 / np.float64(np.float32(sigma) * np.float32(sigma))))
    p1 = np.concatenate([k1[matches[:, 0]].astype(np.float64), np.ones((len(matches), 1))], 1)
    p2 = np.concatenate([k2[matches[:, 1]].astype(np.float64), np.ones((len(matches), 1))], 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        if model == "H":
            Hi = np.stack([np.cross(M[:, 1], M[:, 2]), np.cross(M[:, 2], M[:, 0]), np.cross(M[:, 0], M[:, 1])]) / np.linalg.det(M)
            q = p1 @ M.T
            q = q / q[:, 2:3]
            c1 = ((p2 - q) ** 2).sum(1) * iss
            r = p2 @ Hi.T
            r = r / r[:, 2:3]
            c2 = ((p1 - r) ** 2).sum(1) * iss
        else:
            l2 = p1 @ M.T
            l1 = p2 @ M
            c1 = (l2 * p2).sum(1) ** 2 / (l2[:, 0] ** 2 + l2[:, 1] ** 2) * iss
            c2 = (l1 * p1).sum(1) ** 2 / (l1[:, 0] ** 2 + l1[:, 1] ** 2) * iss
    return c1, c2


def threshold(model):
    return SCORE_THR if model == "H" else CHI_F


def check_inliers(model, M, k1, k2, matches, sigma=1.0):
    """-> (flags, score, (chi1, chi2)): the first direction first; a passing direction adds 5.991 - chi (the first stays when the
    second fails); thr < chi is an outlier"""
    c1, c2 = chis(model, M, k1, k2, matches, sigma)
    thr = threshold(model)
    ok1 = ~(thr < c1)
    ok2 = ok1 & ~(thr < c2)
    score = float(np.where(ok1, SCORE_THR - c1, 0.0).sum() + np.where(ok2, SCORE_THR - c2, 0.0).sum())
    return ok2, score, (c1, c2)
