"""Relocalisation problems for the PnP RANSAC solver (solve::pnp_solver) and an independent numpy float64 restatement of its
arithmetic: the sampler, EPnP (numpy's eigh, lstsq and an SVD Procrustes instead of the Jacobi, Householder and Horn steps)
and check_inliers.  pose = {R row-major (9), t (3)} of cam_pose_cw."""
import numpy as np
from scipy.spatial.transform import Rotation

MIN_SET = 6
GOLDEN = 0x9E3779B97F4A7C15
M64 = 2 ** 64 - 1


def mix(z):
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def sample(seed, k, n, m=MIN_SET):
    """c_j = w_j % (n - j), stepped past the earlier indices in ascending order"""
    out, taken = [], []
    for j in range(m):
        c = mix(seed + GOLDEN * (m * k + j + 1)) % (n - j)
        for a in sorted(taken):
            if c >= a:
                c += 1
        taken.append(c)
        out.append(c)
    return out


def true_pose(rng):
    R = Rotation.from_rotvec(rng.normal(size=3) * 0.7).as_matrix()
    return np.concatenate([R.ravel(), rng.normal(size=3)])


def apply(pose, p):
    return p @ pose[:9].reshape(3, 3).T + pose[9:]


def problem(n, model="perspective", wrong=0.25, noise=0.0, seed=0, planar=False):
    """n correspondences of a frame at a random pose: perspective points 2..10 in front of the camera within a 100 degree cone,
    equirectangular points at 2..10 in every direction (w <= 0 included); `wrong` of them get another landmark's position,
    `noise` is the standard deviation of the bearing's angular noise (radians); planar puts every landmark on one plane."""
    rng = np.random.default_rng(seed)
    pose = true_pose(rng)
    if model == "perspective":
        z = rng.uniform(2.0, 10.0, n)
        pc = np.stack([rng.uniform(-1.0, 1.0, n) * z, rng.uniform(-0.8, 0.8, n) * z, z], 1)
    else:
        d = rng.normal(size=(n, 3))
        pc = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(2.0, 10.0, (n, 1))
    R = pose[:9].reshape(3, 3)
    pw = (pc - pose[9:]) @ R                      # R^T (p_c - t)
    if planar and n:
        # project the landmarks onto the plane through their centroid with a random normal, then re-derive the bearings
        nrm = rng.normal(size=3); nrm /= np.linalg.norm(nrm)
        c = pw.mean(0)
        pw = pw - np.outer((pw - c) @ nrm, nrm)
        pc = apply(pose, pw)
    b = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    if noise > 0.0 and n:
        axis = np.cross(b, rng.normal(size=(n, 3)))
        axis /= np.linalg.norm(axis, axis=1, keepdims=True)
        b = Rotation.from_rotvec(axis * rng.normal(size=(n, 1)) * noise).apply(b)
        b /= np.linalg.norm(b, axis=1, keepdims=True)
    bad = np.zeros(n, bool)
    nb = int(round(wrong * n))
    if nb:
        # a wrong landmark: the true one turned 15..40 degrees about the camera centre, far outside every bound (<= 3.6 degrees)
        sel = rng.choice(n, nb, replace=False)
        bad[sel] = True
        axis = np.cross(pc[sel], rng.normal(size=(nb, 3)))
        axis /= np.linalg.norm(axis, axis=1, keepdims=True)
        moved = Rotation.from_rotvec(axis * np.radians(rng.uniform(15.0, 40.0, (nb, 1)))).apply(pc[sel])
        pw = pw.copy()
        pw[sel] = (moved - pose[9:]) @ R
    octave = rng.integers(0, 8, n)
    sf = (1.2 ** octave).astype(np.float32)
    return dict(bearings=np.ascontiguousarray(b), pos_w=np.ascontiguousarray(pw), scale_factor=sf, pose_true=pose, bad=bad, model=model)


def degenerate(kind, n=40, seed=0):
    """a problem whose first correspondences repeat one landmark (coincident), lie on one line (collinear) or on one plane"""
    p = problem(n, wrong=0.0, seed=seed)
    pw, b = p["pos_w"].copy(), p["bearings"].copy()
    if kind == "coincident":
        pw[:] = pw[0]; b[:] = b[0]
    elif kind == "collinear":
        d = pw[1] - pw[0]
        pw = pw[0] + np.outer(np.linspace(-1.0, 1.0, n), d)
        pc = apply(p["pose_true"], pw)
        b = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    else:
        return problem(n, wrong=0.0, seed=seed, planar=True)
    return dict(p, pos_w=np.ascontiguousarray(pw), bearings=np.ascontiguousarray(b))


def cosines(pose, bearings, pos_w):
    pc = apply(pose, pos_w)
    return (pc * bearings).sum(1) / np.linalg.norm(pc, axis=1)


def max_cos(scale_factor):
    return np.cos(np.pi / 180.0 * np.asarray(scale_factor, np.float32).astype(np.float64))


def check_inliers(pose, p):
    with np.errstate(invalid="ignore", divide="ignore"):
        return cosines(pose, p["bearings"], p["pos_w"]) > max_cos(p["scale_factor"])


def _signed(v):
    return v * (1.0 if v[np.argmax(np.abs(v))] >= 0 else -1.0)


def epnp(bearings, pos_w):
    """EPnP with numpy's eigh / lstsq / SVD: the same conventions as the solver (bearing rows, the eigenvector signs, the sign of
    the camera-frame control points from the first correspondence, the smallest mean (1 - cos) of the three approximations)"""
    b, pw = np.asarray(bearings, np.float64), np.asarray(pos_w, np.float64)
    n = len(b)
    c0 = pw.mean(0)
    d = pw - c0
    lam, U = np.linalg.eigh(d.T @ d)
    cws = [c0] + [c0 + np.sqrt(max(lam[j], 0.0) / n) * _signed(U[:, j]) for j in (2, 1, 0)]
    cws = np.array(cws)
    CC = (cws[1:] - cws[0]).T
    a123 = (np.linalg.inv(CC) @ d.T).T
    al = np.concatenate([1.0 - a123.sum(1, keepdims=True), a123], 1)
    M = np.zeros((2 * n, 12))
    for j in range(4):
        M[0::2, 3 * j] = al[:, j] * b[:, 2]; M[0::2, 3 * j + 2] = -al[:, j] * b[:, 0]
        M[1::2, 3 * j + 1] = al[:, j] * b[:, 2]; M[1::2, 3 * j + 2] = -al[:, j] * b[:, 1]
    _, V = np.linalg.eigh(M.T @ M)
    vs = [_signed(V[:, i]) for i in range(4)]
    pairs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    L = np.zeros((6, 10)); rho = np.zeros(6)
    for j, (a, c) in enumerate(pairs):
        dv = [v[3 * a:3 * a + 3] - v[3 * c:3 * c + 3] for v in vs]
        dd = lambda x, y: float(dv[x] @ dv[y])
        L[j] = [dd(0, 0), 2 * dd(0, 1), dd(1, 1), 2 * dd(0, 2), 2 * dd(1, 2), dd(2, 2), 2 * dd(0, 3), 2 * dd(1, 3), 2 * dd(2, 3), dd(3, 3)]
        rho[j] = np.sum((cws[a] - cws[c]) ** 2)
    best, best_err = None, None
    for ap, cols in ((1, [0, 1, 3, 6]), (2, [0, 1, 2]), (3, [0, 1, 2, 3, 4])):
        x = np.linalg.lstsq(L[:, cols], rho, rcond=None)[0]
        if ap == 1:
            s = -1.0 if x[0] < 0 else 1.0
            b0 = np.sqrt(s * x[0])
            be = np.array([b0, s * x[1] / b0, s * x[2] / b0, s * x[3] / b0])
        else:
            if x[0] < 0:
                b0, b1 = np.sqrt(-x[0]), (np.sqrt(-x[2]) if x[2] < 0 else 0.0)
            else:
                b0, b1 = np.sqrt(x[0]), (np.sqrt(x[2]) if x[2] > 0 else 0.0)
            if x[1] < 0:
                b0 = -b0
            be = np.array([b0, b1, x[3] / b0 if ap == 3 else 0.0, 0.0])
        for _ in range(5):
            B = be
            prod = np.array([B[0] * B[0], B[0] * B[1], B[1] * B[1], B[0] * B[2], B[1] * B[2], B[2] * B[2], B[0] * B[3], B[1] * B[3], B[2] * B[3], B[3] * B[3]])
            J = np.stack([2 * L[:, 0] * B[0] + L[:, 1] * B[1] + L[:, 3] * B[2] + L[:, 6] * B[3],
                          L[:, 1] * B[0] + 2 * L[:, 2] * B[1] + L[:, 4] * B[2] + L[:, 7] * B[3],
                          L[:, 3] * B[0] + L[:, 4] * B[1] + 2 * L[:, 5] * B[2] + L[:, 8] * B[3],
                          L[:, 6] * B[0] + L[:, 7] * B[1] + L[:, 8] * B[2] + 2 * L[:, 9] * B[3]], 1)
            be = be + np.linalg.lstsq(J, rho - L @ prod, rcond=None)[0]
        ccs = sum(be[i] * vs[i] for i in range(4)).reshape(4, 3)
        pcs = al @ ccs
        if pcs[0] @ b[0] < 0:
            pcs = -pcs
        pc0 = pcs.mean(0)
        Hm = (pw - c0).T @ (pcs - pc0)
        U_, _, Vt = np.linalg.svd(Hm)
        D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U_.T))])
        R = Vt.T @ D @ U_.T
        t = pc0 - R @ c0
        pose = np.concatenate([R.ravel(), t])
        err = np.mean(1.0 - cosines(pose, b, pw))
        if best is None or err < best_err:
            best, best_err = pose, err
    return best


def gpu_problem(p):
    return dict(bearings=p["bearings"], pos_w=p["pos_w"], scale_factor=p["scale_factor"])


def args(p):
    return p["bearings"], p["pos_w"], p["scale_factor"]
