"""Loop-closure pose graphs for the graph optimiser's tests, and an independent numpy float64 restatement of one Levenberg
step.  The reference works on 4 x 4 matrices: the edge error is logm(S_ji S_i S_j^-1), the left Jacobian is phi(ad e) read from
the top-right block of expm([[A, I], [0, 0]]), and the damped normal equations are solved with scipy.sparse."""
import numpy as np
import scipy.sparse as sps
import scipy.sparse.linalg as spla
from scipy.linalg import expm, logm
from scipy.spatial.transform import Rotation

from sim3_problems import expm_oplus, from4, generator, to4


def vee(G):
    """sim(3) generator -> (omega, upsilon, sigma)"""
    return np.array([G[2, 1], G[0, 2], G[1, 0], G[0, 3], G[1, 3], G[2, 3], np.trace(G[:3, :3]) / 3.0])


def log4(M):
    return vee(np.real(logm(M)))


def inv4(M):
    return np.linalg.inv(M)


def ad_matrix(xi):
    w, u, s = xi[:3], xi[3:6], xi[6]
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    U = np.array([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]])
    A = np.zeros((7, 7))
    A[:3, :3] = W
    A[3:6, :3] = U
    A[3:6, 3:6] = s * np.eye(3) + W
    A[3:6, 6] = -u
    return A


def Ad_matrix(S):
    R, t, s = np.asarray(S[:9]).reshape(3, 3), np.asarray(S[9:12]), S[12]
    T = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    A = np.zeros((7, 7))
    A[:3, :3] = R
    A[3:6, :3] = T @ R
    A[3:6, 3:6] = s * R
    A[3:6, 6] = -t
    A[6, 6] = 1.0
    return A


def phi(A):
    """(e^A - I) / A from the augmented exponential"""
    n = len(A)
    M = np.zeros((2 * n, 2 * n))
    M[:n, :n] = A
    M[:n, n:] = np.eye(n)
    return expm(M)[:n, n:]


def edge(S_ji, S_i, S_j):
    """e, J_i, J_j of the relative Sim3 edge"""
    E4 = to4(S_ji) @ to4(S_i) @ inv4(to4(S_j))
    e = log4(E4)
    Jl = phi(ad_matrix(e))
    Ji = np.linalg.solve(Jl, Ad_matrix(S_ji))
    Jj = -np.linalg.solve(Jl, Ad_matrix(from4(E4)))
    return e, Ji, Jj


def sim3_of(R, t, s=1.0):
    return np.concatenate([np.asarray(R).ravel(), t, [s]])


def relative(S_j, S_i):
    """S_ji = S_j S_i^-1"""
    return from4(to4(S_j) @ inv4(to4(S_i)))


def loop_graph(num_free, seed=0, fix_scale=False, num_fixed=1, noise=1e-3, drift=(2e-3, 5e-3, 1e-2), cov_step=(2, 3),
               extra_loops=2, num_landmarks=0, fixed_every=0, radius=10.0):
    """A loop trajectory of num_free + num_fixed keyframes on a circle (keyframe 0 fixed: the loop keyframe).
    Edges: spanning-tree parents (k, k+1), covisibilities (k, k + d) for d in cov_step, the loop edge (K-1, 0) and
    extra_loops more near the closure; measurements are the true relative Sim3s times exp(noise).  The start is the chain
    of noisy odometry (rotation, translation, log-scale drift per step; no scale drift with fix_scale).
    fixed_every > 0 fixes every fixed_every-th keyframe as well."""
    rng = np.random.default_rng(seed)
    K = num_free + num_fixed
    true = []
    for k in range(K):
        a = 2 * np.pi * k / K
        R = Rotation.from_rotvec([0, a, 0]).as_matrix() @ Rotation.from_rotvec(rng.normal(size=3) * 0.02).as_matrix()
        c = np.array([radius * np.cos(a), 0.3 * rng.normal(), radius * np.sin(a)])
        true.append(sim3_of(R.T, -R.T @ c, 1.0))        # S_iw: world -> camera
    true = np.array(true)
    pairs = [(k, k + 1) for k in range(K - 1)]
    for d in cov_step:
        pairs += [(k, k + d) for k in range(0, K - d, 1)]
    pairs.append((K - 1, 0))
    for q in range(extra_loops):
        pairs.append((K - 2 - q, q + 1))
    seen, edges = set(), []
    for (i, j) in pairs:
        key = (min(i, j), max(i, j))
        if i == j or min(i, j) < 0 or max(i, j) >= K or key in seen:
            continue
        seen.add(key)
        edges.append((i, j))
    ei = np.array([e[0] for e in edges], np.int32)
    ej = np.array([e[1] for e in edges], np.int32)

    def noisy(S, sig, scale_sig):
        u = rng.normal(size=7) * sig
        u[6] = 0.0 if fix_scale else rng.normal() * scale_sig
        return from4(expm(generator(u)) @ to4(S))

    meas = np.array([noisy(relative(true[j], true[i]), noise, noise) for i, j in zip(ei, ej)])
    # drifted start: odometry along the chain
    start = [true[0].copy()]
    for k in range(1, K):
        u = np.concatenate([rng.normal(size=3) * drift[0], rng.normal(size=3) * drift[1], [0.0 if fix_scale else rng.normal() * drift[2] + 0.5 * drift[2]]])
        rel = from4(expm(generator(u)) @ to4(relative(true[k], true[k - 1])))
        start.append(from4(to4(rel) @ to4(start[-1])))
    start = np.array(start)
    if fix_scale:
        start[:, 12] = 1.0
    fixed = np.zeros(K, np.uint8)
    fixed[:num_fixed] = 1
    if fixed_every:
        fixed[::fixed_every] = 1
    out = dict(true=true, start=start, fixed=fixed, edge_i=ei, edge_j=ej, meas=meas, fix_scale=fix_scale)
    if num_landmarks:
        ref = rng.integers(0, K, size=num_landmarks).astype(np.int32)
        ref[::7] = -1
        pts = rng.normal(size=(num_landmarks, 3)) * 3.0
        out.update(lm=pts, lm_ref=ref)
    return out


def free_index(K, fixed, ei, ej):
    used = np.zeros(K, bool)
    used[ei] = True
    used[ej] = True
    fi = np.full(K, -1)
    free = np.flatnonzero(used & (np.asarray(fixed) == 0))
    fi[free] = np.arange(len(free))
    return fi


def chi2(g, S):
    """sum over the edges of e'e, e = logm(S_ji S_i S_j^-1)"""
    total = 0.0
    for k, (i, j) in enumerate(zip(g["edge_i"], g["edge_j"])):
        e = log4(to4(g["meas"][k]) @ to4(S[i]) @ inv4(to4(S[j])))
        total += float(np.dot(e, e))
    return total


def lm_first_step(g, S, lam=1e-16):
    """The first trial of the first iteration: x of (H + lam I) x = -J'e (sparse solve) and the updated vertices."""
    K = len(S)
    fi = free_index(K, g["fixed"], g["edge_i"], g["edge_j"])
    nf = int(fi.max()) + 1
    n = 7 * nf
    H = sps.lil_matrix((n, n))
    b = np.zeros(n)
    for k, (i, j) in enumerate(zip(g["edge_i"], g["edge_j"])):
        a, c = fi[i], fi[j]
        if a < 0 and c < 0:
            continue
        e, Ji, Jj = edge(g["meas"][k], S[i], S[j])
        blocks = [(a, Ji), (c, Jj)]
        for (u, Ju) in blocks:
            if u < 0:
                continue
            b[7 * u:7 * u + 7] -= Ju.T @ e
            for (w, Jw) in blocks:
                if w >= 0:
                    H[7 * u:7 * u + 7, 7 * w:7 * w + 7] += Ju.T @ Jw
    A = (H.tocsc() + lam * sps.identity(n, format="csc"))
    x = spla.spsolve(A, b)
    out = S.copy()
    for k in range(K):
        if fi[k] >= 0:
            out[k] = expm_oplus(S[k], x[7 * fi[k]:7 * fi[k] + 7], g["fix_scale"])
    return x, out


def pose_of(S):
    """cam_pose_cw = {R, t / s}"""
    S = np.asarray(S).reshape(-1, 13)
    return np.concatenate([S[:, :9], S[:, 9:12] / S[:, 12:13]], axis=1)


def corrected_landmarks(S_init, S_opt, lm, ref):
    out = np.array(lm, np.float64).copy()
    for l, r in enumerate(ref):
        if r < 0:
            continue
        p = np.append(lm[l], 1.0)
        out[l] = (inv4(to4(S_opt[r])) @ to4(S_init[r]) @ p)[:3]
    return out


def trajectory_error(S, true):
    """RMS of the camera-centre errors after aligning vertex 0 (fixed, exact in both)"""
    def centre(x):
        R = x[:9].reshape(3, 3)
        return -R.T @ x[9:12] / x[12]
    return float(np.sqrt(np.mean([np.sum((centre(a) - centre(b)) ** 2) for a, b in zip(S, true)])))
