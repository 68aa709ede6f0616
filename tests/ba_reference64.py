"""A vectorised float64 reference of the optimisers' Levenberg steps, for graphs of any size -- the benchmark's own local BA
(50 free + 10 fixed keyframes, 20 000 landmarks, ~100 000 edges) included.

It restates, in numpy over all edges at once, what tests/ba_graphs.py's reference gets from the oracle edge by edge: the
residuals and Jacobians of the perspective (2-row mono, 3-row stereo) and equirectangular reprojection edges, g2o's SE3
exponential for the pose update, and the Huber weight rho'(chi2).  The damped system is solved by eliminating the points:
the 3 x 3 blocks of Hll + lambda I are inverted as a batch, S = Hpp + lambda I - Hpl (Hll + lambda I)^-1 Hlp is formed
with scipy sparse products, the dense n x n system is solved by LAPACK's Cholesky and the points are back-substituted.
There is no co-observation list, no chunked reduction and no blocked Cholesky of our own, so nothing is shared with the
kernels under test.  (One sparse LU of the full system takes ~30 s at the benchmark's size, and a step makes several
trials: the point elimination keeps a two-iteration reference to seconds.)

The Levenberg driver is `ba_graphs.reference_lm` itself, given this module's `linearise` and `pose_oplus`.
"""
import functools
import os
import sys
from types import SimpleNamespace

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

import ba_graphs as bg


# ------------------------------------------------------------------------------------------------------------ edges
def se3_exp(u):
    """g2o::SE3Quat::exp of updates u (N, 6) = [omega, upsilon]: R (N, 3, 3), t (N, 3).  With Omega = [omega]_x:
    R = I + a Omega + b Omega^2, V = I + b Omega + c Omega^2, t = V upsilon; a, b, c = sin th / th, (1 - cos th) / th^2,
    (th - sin th) / th^3, or their limits 1, 1/2, 1/6 when th < 1e-5 (g2o's switch)."""
    u = np.asarray(u, np.float64).reshape(-1, 6)
    w = u[:, :3]
    th = np.linalg.norm(w, axis=1)
    O = np.zeros((len(u), 3, 3))
    O[:, 0, 1], O[:, 0, 2], O[:, 1, 2] = -w[:, 2], w[:, 1], -w[:, 0]
    O[:, 1, 0], O[:, 2, 0], O[:, 2, 1] = w[:, 2], -w[:, 1], w[:, 0]
    O2 = O @ O
    small = th < 1e-5
    ts = np.where(small, 1.0, th)
    a = np.where(small, 1.0, np.sin(ts) / ts)
    b = np.where(small, 0.5, (1 - np.cos(ts)) / ts ** 2)
    c = np.where(small, 1.0 / 6.0, (ts - np.sin(ts)) / ts ** 3)
    I = np.eye(3)
    R = I + a[:, None, None] * O + b[:, None, None] * O2
    V = I + b[:, None, None] * O + c[:, None, None] * O2
    return R, np.einsum("nij,nj->ni", V, u[:, 3:])


def pose_oplus(poses, u):
    """shot_vertex's update of poses (N, 12) = [R row-major, t]: the estimate becomes exp(u) * estimate"""
    poses = np.asarray(poses, np.float64).reshape(-1, 12)
    Rd, td = se3_exp(u)
    out = np.empty_like(poses)
    out[:, :9] = (Rd @ poses[:, :9].reshape(-1, 3, 3)).reshape(-1, 9)
    out[:, 9:] = np.einsum("nij,nj->ni", Rd, poses[:, 9:]) + td
    return out


def edge_eval(cam, poses, pw, obs, stereo):
    """Residuals e = obs - project(R pw + t) (M, 3) and their Jacobians wrt the pose update [omega, upsilon] (M, 3, 6) and
    the point (M, 3, 3), for M edges at once.  The third row is the stereo x_right row; it is zero on monocular and
    equirectangular edges.  pc = R pw + t moves by -[pc]_x d omega + d upsilon under the update and by R d pw, so each
    Jacobian is -d project / d pc times that."""
    poses = np.asarray(poses, np.float64).reshape(-1, 12)
    R = poses[:, :9].reshape(-1, 3, 3)
    pc = np.einsum("mij,mj->mi", R, pw) + poses[:, 9:]
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    M = len(pc)
    proj = np.zeros((M, 3))
    dproj = np.zeros((M, 3, 3))                      # d project / d pc
    if cam["model"] == "equirectangular":
        L = np.linalg.norm(pc, axis=1)
        xz2 = x * x + z * z
        proj[:, 0] = cam["cols"] * (0.5 + np.arctan2(x, z) / (2 * np.pi))
        proj[:, 1] = cam["rows"] * (0.5 + np.arcsin(y / L) / np.pi)
        cu = cam["cols"] / (2 * np.pi) / xz2
        dproj[:, 0, 0], dproj[:, 0, 2] = cu * z, -cu * x
        cv = cam["rows"] / np.pi / (L * np.sqrt(xz2))       # d asin(y / L) = (L dy - y dL) / (L sqrt(x^2 + z^2))
        dproj[:, 1] = cv[:, None] * (np.array([0.0, 1.0, 0.0]) * L[:, None] - y[:, None] * pc / L[:, None])
        stereo = np.zeros(M, bool)
    else:
        fx, fy, fb = cam["fx"], cam["fy"], cam["focal_x_baseline"]
        proj[:, 0] = fx * x / z + cam["cx"]
        proj[:, 1] = fy * y / z + cam["cy"]
        proj[:, 2] = proj[:, 0] - fb / z
        dproj[:, 0, 0], dproj[:, 0, 2] = fx / z, -fx * x / z ** 2
        dproj[:, 1, 1], dproj[:, 1, 2] = fy / z, -fy * y / z ** 2
        dproj[:, 2] = dproj[:, 0]
        dproj[:, 2, 2] += fb / z ** 2
    stereo = np.asarray(stereo, bool)
    e = np.asarray(obs, np.float64) - proj
    e[~stereo, 2] = 0.0
    dproj[~stereo, 2] = 0.0
    dpc = np.zeros((M, 3, 6))                        # d pc / d [omega, upsilon]
    dpc[:, 0, 1], dpc[:, 0, 2], dpc[:, 1, 2] = z, -y, x
    dpc[:, 1, 0], dpc[:, 2, 0], dpc[:, 2, 1] = -z, y, -x
    dpc[:, :, 3:] = np.eye(3)
    return e, -dproj @ dpc, -dproj @ R


def edges(g, poses, points, xr, idx):
    """edge_eval on the edges `idx` of graph g at the given state"""
    kf, lm = g["obs_kf"][idx], g["obs_lm"][idx]
    obs = np.zeros((len(idx), 3))
    obs[:, :2] = g["obs_xy"][idx]
    stereo = np.zeros(len(idx), bool)
    if xr is not None:
        obs[:, 2] = xr[idx]
        stereo = xr[idx] >= 0
    return edge_eval(g["cam"], poses[kf], points[lm], obs, stereo)


# ----------------------------------------------------------------------------------------------------- the system
def _segment_sum(seg, vals, count):
    """sum of vals (m, ...) per segment id seg (m,) in 0 .. count - 1"""
    k = int(np.prod(vals.shape[1:]))
    flat = (seg[:, None].astype(np.int64) * k + np.arange(k)).ravel()
    return np.bincount(flat, weights=vals.reshape(-1), minlength=count * k).reshape((count,) + vals.shape[1:])


def linearise(g, poses, points, xr, active, delta, with_points):
    """The damped normal equations at the current state, kept in blocks: Hpp (nfree, 6, 6) and bp, Hll (L, 3, 3) and bl,
    Hpl as a sparse n x 3L matrix (edges of one keyframe-landmark pair summed).  Returns the linear system as
    `ba_graphs.reference_lm` takes it (diag, b, free_idx, solve) plus `full(lam)`, the whole damped matrix (sparse)."""
    fixed = g["fixed"]
    free_idx = np.cumsum(fixed == 0) - 1
    free_idx[fixed != 0] = -1
    nfree = int((fixed == 0).sum())
    n, L = 6 * nfree, len(points)
    idx = np.flatnonzero(active)
    e, Jp, Jl = edges(g, poses, points, xr, idx)
    w = g["inv_sigma_sq"][idx].astype(np.float64)
    chi = w * (e * e).sum(1)
    if delta is not None:
        inside = chi <= delta * delta
        w = w * np.where(inside, 1.0, delta / np.sqrt(np.where(inside, 1.0, chi)))
    pf = free_idx[g["obs_kf"][idx]]
    on = pf >= 0
    Hpp = _segment_sum(pf[on], np.einsum("mdi,m,mdj->mij", Jp[on], w[on], Jp[on]), nfree)
    bp = _segment_sum(pf[on], -np.einsum("mdi,m,md->mi", Jp[on], w[on], e[on]), nfree).reshape(-1)
    Hpp_dense = sla.block_diag(*Hpp) if nfree else np.zeros((0, 0))
    if not with_points:
        return SimpleNamespace(diag=np.diagonal(Hpp, axis1=1, axis2=2).reshape(-1), b=bp, free_idx=free_idx,
                               solve=lambda lam: sla.solve(Hpp_dense + lam * np.eye(n), bp, assume_a="pos"),
                               full=lambda lam: sp.csc_matrix(Hpp_dense + lam * np.eye(n)))
    lm = g["obs_lm"][idx]
    Hll = _segment_sum(lm, np.einsum("mdi,m,mdj->mij", Jl, w, Jl), L)
    bl = _segment_sum(lm, -np.einsum("mdi,m,md->mi", Jl, w, e), L)
    Hpl = np.einsum("mdi,m,mdj->mij", Jp[on], w[on], Jl[on])
    rows = np.broadcast_to(6 * pf[on][:, None, None] + np.arange(6)[:, None], Hpl.shape)
    cols = np.broadcast_to(3 * lm[on][:, None, None] + np.arange(3), Hpl.shape)
    W = sp.csr_matrix((Hpl.ravel(), (rows.ravel(), cols.ravel())), shape=(n, 3 * L))

    def solve(lam):
        Dinv = np.linalg.inv(Hll + lam * np.eye(3))
        WD = W @ sp.bsr_matrix((Dinv, np.arange(L), np.arange(L + 1)), shape=(3 * L, 3 * L))
        S = Hpp_dense + lam * np.eye(n) - (WD @ W.T).toarray()
        xp = sla.solve(S, bp - WD @ bl.reshape(-1), assume_a="pos")
        xl = np.einsum("lij,lj->li", Dinv, bl - (W.T @ xp).reshape(L, 3))
        return np.concatenate([xp, xl.reshape(-1)])

    def full(lam):
        Hl = sp.bsr_matrix((Hll, np.arange(L), np.arange(L + 1)), shape=(3 * L, 3 * L))
        return (sp.bmat([[sp.csr_matrix(Hpp_dense), W], [W.T, Hl]]) + lam * sp.identity(n + 3 * L)).tocsc()

    diag = np.concatenate([np.diagonal(Hpp, axis1=1, axis2=2).reshape(-1), np.diagonal(Hll, axis1=1, axis2=2).reshape(-1)])
    return SimpleNamespace(diag=diag, b=np.concatenate([bp, bl.reshape(-1)]), free_idx=free_idx, solve=solve, full=full)


def reference_lm(g, iterations, **kw):
    """ba_graphs.reference_lm's Levenberg driver on this module's linearisation and point-eliminated solve"""
    return bg.reference_lm(None, g, iterations, system=linearise, oplus=pose_oplus, **kw)


# ------------------------------------------------------------------------------------------- the benchmark's problems
def bench_module():
    """the benchmark script, importable from the repository root"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import bench
    return bench


@functools.lru_cache(maxsize=None)
def bench_ba_problem(config):
    """the local-BA problem bench.make_workload builds for rank 0 of --config `config`, with the graph facts the step tests
    check (free_ids, reduced_dim, co_observations)"""
    from openvslam_b200 import synth
    b = bench_module()
    g = synth.ba_problem(b.K_FREE, b.K_FIXED, b.N_LM, model=b.CONFIGS[config]["model"], seed=4)        # make_workload's seed + 4, rank 0
    g["free_ids"] = np.flatnonzero(g["fixed"] == 0)
    g["reduced_dim"] = 6 * len(g["free_ids"])
    g["co_observations"] = bg.co_observations(g)
    return g


@functools.lru_cache(maxsize=None)
def bench_pose_problem(config):
    """the pose-optimiser problem bench.make_workload builds for rank 0 of --config `config`, as a graph of one free
    keyframe whose edge i sees point i (pts_w)"""
    from openvslam_b200 import synth
    b = bench_module()
    cfg = b.CONFIGS[config]
    p = synth.pose_problem(cfg["NKP"], model=cfg["model"], seed=3, stereo=cfg["stereo"])
    M = len(p["obs_kf"])
    return dict(p, points=p["pts_w"].copy(), obs_kf=np.zeros(M, np.int32), obs_lm=np.arange(M, dtype=np.int32),
                fixed=np.zeros(1, np.uint8), free_ids=np.zeros(1, np.int64))


@functools.lru_cache(maxsize=None)
def bench_ba_reference(config):
    """two reference iterations of the benchmark's local BA (lambda_init, trials, states)"""
    return reference_lm(bench_ba_problem(config), 2)[2]


@functools.lru_cache(maxsize=None)
def bench_pose_reference(config):
    """one reference iteration of the benchmark's pose problem (points constant)"""
    return reference_lm(bench_pose_problem(config), 1, with_points=False)[2]


def pair_chunks(g, chunk=128):
    """(number of free-keyframe pairs with a co-observation, diagonal included; the fewest 128-record chunks of a diagonal
    pair; the most records of an off-diagonal pair)"""
    on = g["fixed"][g["obs_kf"]] == 0
    free_idx = np.cumsum(g["fixed"] == 0) - 1
    kf, lm = free_idx[g["obs_kf"][on]], g["obs_lm"][on]
    nfree = int((g["fixed"] == 0).sum())
    A = sp.csr_matrix((np.ones(len(kf)), (kf, lm)), shape=(nfree, len(g["points"])))
    C = (A @ A.T).toarray()
    off = C[np.triu_indices(nfree, 1)]
    return int((np.triu(C) > 0).sum()), int(-(-np.diag(C).min() // chunk)), int(off.max())
