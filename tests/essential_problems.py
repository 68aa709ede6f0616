"""Two-view problems for the essential-matrix RANSAC solver (solve::essential_solver) and an independent numpy float64 restatement
of its arithmetic: the eight-point E_21 with numpy's SVD on A (not the Jacobi on A^T A) and an SVD rank-2 projection, and
check_inliers.  A match is a pair of unit bearings (b1 in camera 1, b2 in camera 2); b2^T E_21 b1 = 0 with E_21 = [t_21]x R_21,
p_2 = R_21 p_1 + t_21."""
import numpy as np
from scipy.spatial.transform import Rotation

from pnp_problems import sample as _sample

MIN_SET = 8
THR = 0.01745240643


def sample(seed, k, n):
    return _sample(seed, k, n, MIN_SET)


def skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def true_E(R, t):
    return skew(t) @ R


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def problem(n, model="perspective", wrong=0.25, noise=0.0, seed=0, planar=False, pure_rotation=False):
    """n matches between camera 1 (the origin) and camera 2 (R_21, t_21): perspective points 2..10 in front of camera 1 within a
    90 degree cone and a small motion, equirectangular points at 2..10 in every direction (w <= 0 included) and a larger one;
    `wrong` of the matches get a camera-2 bearing turned 5..30 degrees off its epipolar plane; `noise` is the standard deviation of
    both bearings' angular noise (radians); planar puts every point on one plane; pure_rotation sets t = 0."""
    rng = np.random.default_rng(seed)
    if model == "perspective":
        R = Rotation.from_rotvec(rng.normal(size=3) * 0.2).as_matrix()
        t = rng.normal(size=3) * 0.6
        z = rng.uniform(2.0, 10.0, n)
        p1 = np.stack([rng.uniform(-1.0, 1.0, n) * z, rng.uniform(-0.8, 0.8, n) * z, z], 1)
    else:
        R = Rotation.from_rotvec(rng.normal(size=3) * 0.7).as_matrix()
        t = rng.normal(size=3)
        p1 = _unit(rng.normal(size=(n, 3))) * rng.uniform(2.0, 10.0, (n, 1))
    if pure_rotation:
        t = np.zeros(3)
    if planar and n:
        nrm = _unit(rng.normal(size=3))
        c = p1.mean(0)
        p1 = p1 - np.outer((p1 - c) @ nrm, nrm)
    p2 = p1 @ R.T + t
    b1, b2 = _unit(p1), _unit(p2)

    def jitter(b):
        axis = _unit(np.cross(b, rng.normal(size=b.shape)))
        return _unit(Rotation.from_rotvec(axis * rng.normal(size=(len(b), 1)) * noise).apply(b))
    if noise > 0.0 and n:
        b1, b2 = jitter(b1), jitter(b2)
    bad = np.zeros(n, bool)
    nb = int(round(wrong * n))
    if nb and not pure_rotation:
        sel = rng.choice(n, nb, replace=False)
        bad[sel] = True
        E = true_E(R, t)
        nrm = _unit((b1[sel] @ E.T))                  # the normal of each epipolar plane in camera 2
        ang = np.radians(rng.uniform(5.0, 30.0, (nb, 1))) * rng.choice([-1.0, 1.0], (nb, 1))
        inplane = _unit(b2[sel] - (b2[sel] * nrm).sum(1, keepdims=True) * nrm)
        b2 = b2.copy()
        b2[sel] = _unit(np.cos(ang) * inplane + np.sin(ang) * nrm)
    return dict(bearings_1=np.ascontiguousarray(b1), bearings_2=np.ascontiguousarray(b2), R=R, t=t, E_true=true_E(R, t), bad=bad,
                model=model)


def degenerate(kind, n=40, seed=0):
    """coincident (every match the same pair), collinear (points on one line through space), planar, or pure rotation"""
    if kind == "planar":
        return problem(n, wrong=0.0, seed=seed, planar=True)
    if kind == "rotation":
        return problem(n, wrong=0.0, seed=seed, pure_rotation=True)
    p = problem(n, wrong=0.0, seed=seed)
    b1, b2 = p["bearings_1"].copy(), p["bearings_2"].copy()
    if kind == "coincident":
        b1[:] = b1[0]; b2[:] = b2[0]
    else:   # collinear
        rng = np.random.default_rng(seed + 1)
        a, d = np.array([0.0, 0.0, 5.0]), _unit(rng.normal(size=3))
        p1 = a + np.outer(np.linspace(-1.0, 1.0, n), d)
        p2 = p1 @ p["R"].T + p["t"]
        b1, b2 = _unit(p1), _unit(p2)
    return dict(p, bearings_1=np.ascontiguousarray(b1), bearings_2=np.ascontiguousarray(b2))


def canonical(E):
    """the sign convention: the entry of largest magnitude (first on ties) positive"""
    f = E.ravel()
    return E * (-1.0 if f[np.argmax(np.abs(f))] < 0 else 1.0)


def compute_E(b1, b2):
    """the eight-point E_21: the right singular vector of A's smallest singular value, then U diag(s, s, 0) V^T with s the mean of
    the two largest singular values"""
    A = np.einsum("ni,nj->nij", np.asarray(b2), np.asarray(b1)).reshape(-1, 9)
    e = np.linalg.svd(A)[2][-1]
    U, S, Vt = np.linalg.svd(e.reshape(3, 3))
    s = (S[0] + S[1]) / 2.0
    return canonical(U @ np.diag([s, s, 0.0]) @ Vt)


def residuals(E, b1, b2):
    """(r2, r1) per match"""
    e1 = b1 @ E.T
    e2 = b2 @ E
    with np.errstate(invalid="ignore", divide="ignore"):
        r2 = np.abs((e1 * b2).sum(1)) / np.linalg.norm(e1, axis=1)
        r1 = np.abs((e2 * b1).sum(1)) / np.linalg.norm(e2, axis=1)
    return r2, r1


def check_inliers(E, b1, b2):
    """-> (flags, score): r2 first, then r1; the passing residuals join the score (r2 stays when r1 fails); !(thr < r)"""
    r2, r1 = residuals(E, b1, b2)
    ok2 = ~(THR < r2)
    ok1 = ok2 & ~(THR < r1)
    return ok1, float(np.where(ok2, r2, 0.0).sum() + np.where(ok1, r1, 0.0).sum())


def gpu_problem(p):
    return dict(bearings_1=p["bearings_1"], bearings_2=p["bearings_2"])
