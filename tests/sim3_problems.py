"""Loop-closure problems for the transform optimiser (optimize::transform_optimizer) and a float64 numpy restatement of one of
its Levenberg iterations that shares no code with the oracle: numpy projection and Jacobians, scipy's expm for the update, a
dense 7 x 7 damped solve with the fixed-scale rule (the solve stays 7 x 7, update[6] is zeroed before the exponential).

sim3 = {R row-major (9), t (3), s}, S p = s R p + t, maps keyframe 2's camera frame into keyframe 1's."""
import numpy as np
from scipy.linalg import expm
from scipy.spatial.transform import Rotation

CAMS = {
    "perspective": dict(model="perspective", fx=520.0, fy=515.0, cx=320.0, cy=240.0, cols=640.0, rows=480.0),
    "equirectangular": dict(model="equirectangular", cols=1920.0, rows=960.0),
}


def skew(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])


def generator(u):
    G = np.zeros((4, 4))
    G[:3, :3] = u[6] * np.eye(3) + skew(u[:3])
    G[:3, 3] = u[3:6]
    return G


def to4(S):
    M = np.eye(4)
    M[:3, :3] = S[12] * np.asarray(S[:9]).reshape(3, 3)
    M[:3, 3] = S[9:12]
    return M


def from4(M):
    s = np.cbrt(np.linalg.det(M[:3, :3]))
    return np.concatenate([(M[:3, :3] / s).ravel(), M[:3, 3], [s]])


def expm_oplus(S, u, fix_scale):
    u = np.array(u, np.float64)
    if fix_scale:
        u[6] = 0.0
    out = from4(expm(generator(u)) @ to4(S))
    if fix_scale:
        out[12] = S[12]
    return out


def _pose(rng, angle, trans):
    R = Rotation.from_rotvec(rng.normal(size=3) * angle).as_matrix()
    return np.concatenate([R.ravel(), rng.normal(size=3) * trans])


def project(cam, p):
    """pixels (N, 2) and d pixel / d p (N, 2, 3)"""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    P = np.zeros((len(p), 2, 3))
    if cam["model"] == "equirectangular":
        L = np.sqrt(x * x + y * y + z * z)
        uv = np.stack([cam["cols"] * (0.5 + np.arctan2(x, z) / (2 * np.pi)), cam["rows"] * (0.5 + np.arcsin(y / L) / np.pi)], 1)
        xz2 = x * x + z * z
        P[:, 0, 0] = cam["cols"] / (2 * np.pi) * z / xz2
        P[:, 0, 2] = -cam["cols"] / (2 * np.pi) * x / xz2
        # d asin(y / L) = (e_y / L - y p / L^3) / sqrt(1 - y^2 / L^2)
        k = cam["rows"] / np.pi / np.sqrt(1 - (y / L) ** 2)
        P[:, 1, :] = (k / L)[:, None] * (np.eye(3)[1][None, :] - (y / L ** 2)[:, None] * p)
        return uv, P
    uv = np.stack([cam["fx"] * x / z + cam["cx"], cam["fy"] * y / z + cam["cy"]], 1)
    P[:, 0, 0] = cam["fx"] / z
    P[:, 0, 2] = -cam["fx"] * x / z ** 2
    P[:, 1, 1] = cam["fy"] / z
    P[:, 1, 2] = -cam["fy"] * y / z ** 2
    return uv, P


def problem(n, model="perspective", fix_scale=False, wrong=0.15, noise=1.0, perturb=(0.01, 0.05, 0.02), seed=0, num_good=None):
    """Two keyframes with a known S_12 (scale 1.35 unless fix_scale), n correspondences with pixel noise `noise`, a fraction
    `wrong` of them (or all but `num_good`) moved far off in keyframe 1, and a start exp(perturbation) S_12."""
    rng = np.random.default_rng(seed)
    cam = CAMS[model]
    S_true = np.concatenate([Rotation.from_rotvec([0.02, 0.15, -0.03]).as_matrix().ravel(), [0.4, -0.1, 0.25],
                             [1.0 if fix_scale else 1.35]])
    pose_1w, pose_2w = _pose(rng, 0.8, 1.0), _pose(rng, 0.8, 1.0)
    pc2 = []
    while sum(len(a) for a in pc2) < n:
        m = 4 * n + 16
        if model == "equirectangular":
            d = rng.normal(size=(m, 3))
            p = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(2, 10, (m, 1))
        else:
            z = rng.uniform(3, 12, m)
            p = np.stack([rng.uniform(-0.55, 0.55, m) * z, rng.uniform(-0.4, 0.4, m) * z, z], 1)
        q = S_true[12] * p @ S_true[:9].reshape(3, 3).T + S_true[9:12]
        keep = np.ones(m, bool)
        if model == "perspective":
            uv1, _ = project(cam, q)
            keep = (q[:, 2] > 1.0) & (uv1[:, 0] > 5) & (uv1[:, 0] < 635) & (uv1[:, 1] > 5) & (uv1[:, 1] < 475)
        pc2.append(p[keep])
    pc2 = np.concatenate(pc2)[:n]
    pc1 = S_true[12] * pc2 @ S_true[:9].reshape(3, 3).T + S_true[9:12]

    def world(pose, pc):
        R = pose[:9].reshape(3, 3)
        return (pc - pose[9:12]) @ R                       # R^T (pc - t), row-wise
    levels_1, levels_2 = rng.integers(0, 8, n), rng.integers(0, 8, n)
    sig1, sig2 = 1.2 ** levels_1, 1.2 ** levels_2
    obs1 = project(cam, pc1)[0] + rng.normal(size=(n, 2)) * noise * sig1[:, None]
    obs2 = project(cam, pc2)[0] + rng.normal(size=(n, 2)) * noise * sig2[:, None]
    num_wrong = int(round(wrong * n)) if num_good is None else n - num_good
    bad = rng.permutation(n)[:num_wrong]
    ang = rng.uniform(0, 2 * np.pi, num_wrong)
    obs1[bad] += np.stack([np.cos(ang), np.sin(ang)], 1) * rng.uniform(40, 120, (num_wrong, 1))
    if model == "equirectangular":
        obs1[:, 0] %= cam["cols"]
    du = np.concatenate([rng.normal(size=3) * perturb[0], rng.normal(size=3) * perturb[1], [0.0 if fix_scale else perturb[2]]])
    S0 = expm_oplus(S_true, du, False)
    if fix_scale:
        S0[12] = 1.0
    inv1 = (1.0 / sig1 ** 2).astype(np.float32)
    inv2 = (1.0 / sig2 ** 2).astype(np.float32)
    return dict(cam=cam, model=model, fix_scale=fix_scale, S_true=S_true, S0=S0, pose_1w=pose_1w, pose_2w=pose_2w,
                pos_w_1=world(pose_1w, pc1), obs_xy_1=obs1.astype(np.float32), inv_sigma_sq_1=inv1,
                pos_w_2=world(pose_2w, pc2), obs_xy_2=obs2.astype(np.float32), inv_sigma_sq_2=inv2, bad=np.sort(bad))


def args(p):
    """positional arguments after the two cameras, as the optimisers take them"""
    return (p["pose_1w"], p["pose_2w"], p["pos_w_1"], p["obs_xy_1"], p["inv_sigma_sq_1"], p["pos_w_2"], p["obs_xy_2"],
            p["inv_sigma_sq_2"], p["S0"])


# ---------------------------------------------------------------------------------------------- numpy reference
def camera_points(p):
    R1, R2 = p["pose_1w"][:9].reshape(3, 3), p["pose_2w"][:9].reshape(3, 3)
    return p["pos_w_1"] @ R1.T + p["pose_1w"][9:12], p["pos_w_2"] @ R2.T + p["pose_2w"][9:12]


def residuals(p, S, jacobians=False):
    """e12 (n, 2), e21 (n, 2) and, if asked, their Jacobians (n, 2, 7) with respect to S <- exp(xi) S"""
    pc1, pc2 = camera_points(p)
    R, t, s = S[:9].reshape(3, 3), S[9:12], S[12]
    q1 = s * pc2 @ R.T + t
    q2 = (pc1 - t) @ R / s
    uv1, P1 = project(p["cam"], q1)
    uv2, P2 = project(p["cam"], q2)
    e12 = p["obs_xy_1"].astype(np.float64) - uv1
    e21 = p["obs_xy_2"].astype(np.float64) - uv2
    if not jacobians:
        return e12, e21
    n = len(pc1)
    D1 = np.zeros((n, 3, 7))
    D1[:, :, :3] = -np.array([skew(v) for v in q1])
    D1[:, :, 3:6] = np.eye(3)
    D1[:, :, 6] = q1
    M = np.zeros((n, 3, 7))
    M[:, :, :3] = np.array([skew(v) for v in pc1])
    M[:, :, 3:6] = -np.eye(3)
    M[:, :, 6] = -pc1
    D2 = np.einsum("ji,njk->nik", R, M) / s
    return e12, e21, -np.einsum("nij,njk->nik", P1, D1), -np.einsum("nij,njk->nik", P2, D2)


def _robust(chi, delta):
    rho0 = np.where(chi <= delta * delta, chi, 2 * np.sqrt(chi) * delta - delta * delta)
    rho1 = np.where(chi <= delta * delta, 1.0, delta / np.sqrt(np.maximum(chi, 1e-300)))
    return rho0, rho1


def robust_chi2(p, S, delta, active):
    e12, e21 = residuals(p, S)
    c12 = p["inv_sigma_sq_1"].astype(np.float64) * (e12 ** 2).sum(1)
    c21 = p["inv_sigma_sq_2"].astype(np.float64) * (e21 ** 2).sum(1)
    return float((_robust(c12, delta)[0] + _robust(c21, delta)[0])[active].sum())


def system(p, S, delta, active):
    e12, e21, J12, J21 = residuals(p, S, True)
    H = np.zeros((7, 7)); b = np.zeros(7)
    for e, J, w in ((e12, J12, p["inv_sigma_sq_1"]), (e21, J21, p["inv_sigma_sq_2"])):
        w = w.astype(np.float64)
        ww = _robust(w * (e ** 2).sum(1), delta)[1] * w
        e, J, ww = e[active], J[active], ww[active]
        H += np.einsum("nik,n,nil->kl", J, ww, J)
        b -= np.einsum("nik,n,ni->k", J, ww, e)
    return H, b


def lm_iteration(p, S, delta, active=None):
    """g2o's first Levenberg iteration from S -> (S after it, trials, lambda_init)"""
    active = np.ones(len(p["inv_sigma_sq_1"]), bool) if active is None else active
    chi0 = robust_chi2(p, S, delta, active)
    H, b = system(p, S, delta, active)
    lam = 1e-5 * np.abs(np.diag(H)).max()
    lam0, ni = lam, 2.0
    for q in range(1, 11):
        x = np.linalg.solve(H + lam * np.eye(7), b)           # 7 x 7 whatever the scale mode
        Sn = expm_oplus(S, x, p["fix_scale"])
        chi1 = robust_chi2(p, Sn, delta, active)
        rho = (chi0 - chi1) / (x @ (lam * x + b) + 1e-3)
        if rho > 0 and np.isfinite(chi1):
            return Sn, q, lam0
        lam *= ni
        ni *= 2
    return S, 10, lam0


def step_error(x, x_ref, x_start):
    x, x_ref, x_start = (np.asarray(a, np.float64) for a in (x, x_ref, x_start))
    return float(np.abs(x - x_ref).max() / np.abs(x_ref - x_start).max())
