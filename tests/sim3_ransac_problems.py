"""Loop-detection problems for the Sim3 RANSAC solver (solve::sim3_solver), built on tests/sim3_problems.py's keyframe pairs, and a
vectorised numpy float64 restatement of the sampler and of count_inliers that shares no code with the oracle.

A problem holds two keyframes related by a known S_12 and n landmark pairs; a fraction `wrong` of them are wrong 3-D
correspondences (keyframe 1's landmark moved by ~1.5 m)."""
import numpy as np

import sim3_problems as sp

GOLDEN = 0x9E3779B97F4A7C15
MASK = (1 << 64) - 1
CHI_SQ_2D = np.float32(9.21034)


def _world(pose, pc):
    return (pc - pose[9:12]) @ pose[:9].reshape(3, 3)


def problem(n, model="perspective", fix_scale=False, wrong=0.25, noise3d=0.0, seed=0, behind=0):
    """n pairs; `noise3d` adds that much (m) Gaussian noise to keyframe 1's landmarks; `behind` pairs get keyframe 2's landmark
    behind camera 2 (perspective)."""
    rng = np.random.default_rng(1000 + seed)
    p = sp.problem(max(n, 3), model=model, fix_scale=fix_scale, wrong=0.0, seed=seed)
    pos_w_1, pos_w_2 = p["pos_w_1"][:n].copy(), p["pos_w_2"][:n].copy()
    sig1 = (np.float32(1.0) / p["inv_sigma_sq_1"][:n]).astype(np.float32)
    sig2 = (np.float32(1.0) / p["inv_sigma_sq_2"][:n]).astype(np.float32)
    if noise3d:
        pos_w_1 += rng.normal(size=pos_w_1.shape) * noise3d
    bad = np.sort(rng.permutation(n)[:int(round(wrong * n))])
    pos_w_1[bad] += rng.normal(size=(len(bad), 3)) * 1.5
    if behind:
        R2 = p["pose_2w"][:9].reshape(3, 3)
        idx = rng.permutation(n)[:behind]
        pc2 = pos_w_2[idx] @ R2.T + p["pose_2w"][9:12]
        pos_w_2[idx] = _world(p["pose_2w"], -pc2)
    return dict(cam=p["cam"], model=model, fix_scale=fix_scale, S_true=p["S_true"], pose_1w=p["pose_1w"], pose_2w=p["pose_2w"],
                pos_w_1=pos_w_1, sigma_sq_1=sig1, pos_w_2=pos_w_2, sigma_sq_2=sig2, bad=bad)


def degenerate(kind, model="perspective", fix_scale=False, seed=0):
    """three pairs whose keyframe-2 points (and so keyframe-1 points) coincide or lie on one line"""
    p = problem(3, model=model, fix_scale=fix_scale, wrong=0.0, seed=seed)
    S = p["S_true"]
    R2 = p["pose_2w"][:9].reshape(3, 3)
    pc2 = p["pos_w_2"] @ R2.T + p["pose_2w"][9:12]
    if kind == "coincident":
        pc2[1] = pc2[0]; pc2[2] = pc2[0]
    else:
        pc2[2] = 2.0 * pc2[1] - pc2[0]
    pc1 = S[12] * pc2 @ S[:9].reshape(3, 3).T + S[9:12]
    p["pos_w_2"] = _world(p["pose_2w"], pc2)
    p["pos_w_1"] = _world(p["pose_1w"], pc1)
    return p


def args(p):
    """positional arguments after the two cameras, as the oracle takes them"""
    return p["pose_1w"], p["pose_2w"], p["pos_w_1"], p["sigma_sq_1"], p["pos_w_2"], p["sigma_sq_2"]


def gpu_problem(p):
    from openvslam_b200 import optimize
    cam = optimize.camera(**p["cam"])
    return dict(cam_1=cam, cam_2=cam, pose_1w=p["pose_1w"], pose_2w=p["pose_2w"], pos_w_1=p["pos_w_1"], sigma_sq_1=p["sigma_sq_1"],
                pos_w_2=p["pos_w_2"], sigma_sq_2=p["sigma_sq_2"])


# ---------------------------------------------------------------------------------------------- numpy restatement
def mix(z):
    z &= MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def triple(seed, k, n):
    w = [mix(seed + GOLDEN * (3 * k + j + 1)) for j in range(3)]
    i0 = w[0] % n
    c = w[1] % (n - 1)
    i1 = c + (c >= i0)
    i2 = w[2] % (n - 2)
    for m in sorted((i0, i1)):
        if i2 >= m:
            i2 += 1
    return [int(i0), int(i1), int(i2)]


def camera_points(p):
    R1, R2 = p["pose_1w"][:9].reshape(3, 3), p["pose_2w"][:9].reshape(3, 3)
    return p["pos_w_1"] @ R1.T + p["pose_1w"][9:12], p["pos_w_2"] @ R2.T + p["pose_2w"][9:12]


def reproject(cam, pc):
    """(uv (N, 2), in front (N,)) of camera-frame points"""
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    if cam["model"] == "equirectangular":
        L = np.sqrt(x * x + y * y + z * z)
        lon = np.arctan2(x / L, z / L)
        lat = -np.arcsin(y / L)
        return np.stack([cam["cols"] * (0.5 + lon / (2 * np.pi)), cam["rows"] * (0.5 - lat / np.pi)], 1), np.ones(len(pc), bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = np.stack([cam["fx"] * x / z + cam["cx"], cam["fy"] * y / z + cam["cy"]], 1)
    return uv, z > 0


def horn_eigh(p1, p2, fix_scale):
    """Horn's solution with numpy's eigh -> S12 (R, t, s)"""
    A1, A2 = (p1 - p1.mean(0)).T, (p2 - p2.mean(0)).T
    M = A2 @ A1.T
    (Sxx, Sxy, Sxz), (Syx, Syy, Syz), (Szx, Szy, Szz) = M
    N = np.array([[Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx], [Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz],
                  [Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy], [Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz]])
    w, x, y, z = np.linalg.eigh(N)[1][:, -1]
    R = np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])
    s = 1.0 if fix_scale else float(np.sum(A1 * (R @ A2)) / np.sum(A2 * A2))
    t = p1.mean(0) - s * R @ p2.mean(0)
    return np.concatenate([R.ravel(), t, [s]])


def umeyama(p1, p2, fix_scale):
    """the least-squares similarity p1 ~ s R p2 + t by SVD (Umeyama) -> S12"""
    c1, c2 = p1.mean(0), p2.mean(0)
    A1, A2 = p1 - c1, p2 - c2
    U, D, Vt = np.linalg.svd(A1.T @ A2)
    E = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = U @ E @ Vt
    s = 1.0 if fix_scale else float(np.trace(np.diag(D) @ E) / np.sum(A2 * A2))
    return np.concatenate([R.ravel(), c1 - s * R @ c2, [s]])


def errors(p, S12):
    """(e1 (n,), e2 (n,), ok (n,), bound1, bound2) of count_inliers for S12: squared reprojection errors in keyframe 1 and 2"""
    pc1, pc2 = camera_points(p)
    R, t, s = S12[:9].reshape(3, 3), S12[9:12], S12[12]
    r1, ok1 = reproject(p["cam"], pc1)
    r2, ok2 = reproject(p["cam"], pc2)
    u2, f2 = reproject(p["cam"], (pc1 - t) @ R / s)          # S_21 pc1
    u1, f1 = reproject(p["cam"], s * pc2 @ R.T + t)          # S_12 pc2
    e2 = ((u2 - r2) ** 2).sum(1)
    e1 = ((u1 - r1) ** 2).sum(1)
    b1 = (CHI_SQ_2D * p["sigma_sq_1"]).astype(np.float32).astype(np.float64)
    b2 = (CHI_SQ_2D * p["sigma_sq_2"]).astype(np.float32).astype(np.float64)
    return e1, e2, ok1 & ok2 & f1 & f2, b1, b2


def count_inliers(p, S12):
    e1, e2, ok, b1, b2 = errors(p, S12)
    with np.errstate(invalid="ignore"):
        return ok & (e1 < b1) & (e2 < b2)
