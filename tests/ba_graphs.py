"""Bundle-adjustment graphs with a chosen structure, and an independent float64 Levenberg step to compare the optimisers with.

`graph()` returns problems in the dict layout of `openvslam_b200.synth.ba_problem` (which stays the benchmark's generator), but
lets a test choose what `synth` never produces: where the fixed keyframes sit (so that a keyframe's index in the reduced system
differs from its id), the exact number of co-observations of chosen keyframe pairs, free keyframes without observations,
landmarks without observations or seen only from fixed keyframes, single-view mono landmarks, one landmark seen by every free
keyframe, monocular keyframes in a stereo setup and landmarks behind the cameras.  Seeded, pure numpy.

`reference_lm()` runs g2o's Levenberg iterations (lambda_0 = 1e-5 max diag, rho test, lambda schedule, <= 10 trials) on the FULL
normal equations over poses and points -- no Schur complement, no Cholesky of our own: scipy's sparse LU -- with the per-edge
residuals and Jacobians of `oracle.edge_eval` (pinned against finite differences) and the Huber weights rho'(chi2) at the
linearisation point.  It shares no linear algebra with the oracle's Schur / Cholesky path or with the kernels.
"""
import functools
from types import SimpleNamespace

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from openvslam_b200 import synth

CHI2_2D, CHI2_3D = 5.99146, 7.81473

PERSPECTIVE = dict(model="perspective", fx=718.856, fy=718.856, cx=607.19, cy=185.21, focal_x_baseline=386.1448, cols=1241.0, rows=376.0)
EQUIRECTANGULAR = dict(model="equirectangular", fx=0.0, fy=0.0, cx=0.0, cy=0.0, focal_x_baseline=0.0, cols=1920.0, rows=960.0)


def fixed_mask(num_free, num_fixed, pattern="last"):
    """Fixed flags of K = num_free + num_fixed keyframes: the fixed ones "first", "last", or "interleaved" (spread evenly over
    the ids, starting with keyframe 0: num_fixed = K / 3 fixes every third keyframe)."""
    K = num_free + num_fixed
    fixed = np.zeros(K, np.uint8)
    if pattern == "first":
        fixed[:num_fixed] = 1
    elif pattern == "last":
        fixed[num_free:] = 1
    elif pattern == "interleaved":
        fixed[(np.arange(num_fixed) * K) // max(num_fixed, 1)] = 1
    else:
        raise ValueError(pattern)
    assert int(fixed.sum()) == num_fixed
    return fixed


def graph(num_free, num_fixed=0, fixed="last", num_landmarks=200, views=(2, 5), pair_counts=None, empty_free=(), unobserved=0,
          fixed_only=0, single_view=0, seen_by_all=0, behind=0, seam=0, mono_keyframes=(), stereo=False, model="perspective", seed=0,
          pixel_sigma=1.0, outlier_frac=0.05, pose_noise=(0.01, 0.05), point_noise=0.05):
    """A local-BA problem.  Free keyframes are addressed by their ordinal among the free ones (0 .. num_free - 1), other
    keyframe arguments by id.

    num_landmarks   landmarks seen by `views` = (lo, hi) random keyframes (free or fixed, never an empty free keyframe);
    pair_counts     {(a, b): c}: c more landmarks seen by exactly the free keyframes a and b (and possibly one fixed keyframe).
                    A random landmark then sees at most one of the keyframes named here, so pair (a, b) has exactly c
                    co-observations;
    empty_free      free keyframes without any observation;
    unobserved      landmarks without observations: the first one, the last one, the rest at random positions;
    fixed_only      landmarks seen by two fixed keyframes only;
    single_view     landmarks seen by one free keyframe through a monocular edge (rank-2 Hll);
    seen_by_all     landmarks seen by every (non-empty) free keyframe;
    behind          landmarks behind every camera (negative depth: classified as outliers after round 1, perspective only);
    seam            equirectangular landmarks estimated across the longitude seam from where they are observed (appended last):
                    the first Levenberg iterations need several trials;
    mono_keyframes  keyframe ids whose edges are monocular in a stereo setup.
    Observations are grouped by landmark and every (keyframe, landmark) pair occurs at most once."""
    rng = np.random.default_rng(seed)
    K = num_free + num_fixed
    cam = dict(EQUIRECTANGULAR if model == "equirectangular" else PERSPECTIVE)
    stereo = bool(stereo) and model != "equirectangular"
    fx = fixed_mask(num_free, num_fixed, fixed)
    free_ids = np.flatnonzero(fx == 0)
    fixed_ids = np.flatnonzero(fx)
    empty = set(int(free_ids[a]) for a in empty_free)
    live_free = [int(k) for k in free_ids if int(k) not in empty]
    eligible = np.array(live_free + [int(k) for k in fixed_ids])
    designated = set()
    for a, b in (pair_counts or {}):
        designated |= {int(free_ids[a]), int(free_ids[b])}

    # keyframes in a 2 m x 0.6 m x 2 m box looking down +z, landmarks 5-15 m ahead: every camera sees every landmark in front
    poses = np.zeros((K, 12))
    for k in range(K):
        c = rng.uniform([-1.0, -0.3, -1.0], [1.0, 0.3, 1.0])
        R = synth._rot(0.05 * rng.standard_normal(3))
        poses[k, :9] = R.reshape(-1); poses[k, 9:] = -R @ c

    view_sets, mono_lm = [], []
    for _ in range(num_landmarks):
        m = int(rng.integers(views[0], views[1] + 1))
        kfs = [int(k) for k in rng.choice(eligible, size=min(m, len(eligible)), replace=False)]
        seen = [k for k in kfs if k in designated]
        kfs = [k for k in kfs if k not in designated or k == (seen[0] if seen else None)]
        view_sets.append(kfs); mono_lm.append(False)
    for (a, b), c in (pair_counts or {}).items():
        for _ in range(c):
            kfs = [int(free_ids[a]), int(free_ids[b])]
            if len(fixed_ids) and rng.random() < 0.5:
                kfs.append(int(rng.choice(fixed_ids)))
            view_sets.append(kfs); mono_lm.append(False)
    for _ in range(fixed_only):
        view_sets.append([int(k) for k in rng.choice(fixed_ids, size=min(2, len(fixed_ids)), replace=False)]); mono_lm.append(False)
    for _ in range(single_view):
        view_sets.append([int(rng.choice(live_free))]); mono_lm.append(True)
    for _ in range(seen_by_all):
        view_sets.append(list(live_free)); mono_lm.append(False)
    is_behind = [False] * len(view_sets)
    for _ in range(behind):
        view_sets.append([int(k) for k in rng.choice(live_free, size=min(2, len(live_free)), replace=False)]); mono_lm.append(False)
        is_behind.append(True)
    order = rng.permutation(len(view_sets))
    view_sets = [sorted(view_sets[i]) for i in order]
    mono_lm = [mono_lm[i] for i in order]
    is_behind = [is_behind[i] for i in order]
    if unobserved:
        L = len(view_sets) + unobserved
        gaps = [0, L - 1][:unobserved]
        gaps += sorted(int(x) + 1 for x in rng.choice(L - 2, size=unobserved - len(gaps), replace=False)) if unobserved > 2 else []
        gaps = sorted(set(gaps))
        assert len(gaps) == unobserved
        for q in gaps:
            view_sets.insert(q, []); mono_lm.insert(q, False); is_behind.insert(q, False)
    L = len(view_sets)

    z = rng.uniform(5, 15, L)
    points = np.stack([rng.uniform(-0.4, 0.4, L) * z, rng.uniform(-0.25, 0.25, L) * z, z], 1)
    points[np.array(is_behind, bool), 2] *= -1.0
    mono_kf = np.zeros(K, bool); mono_kf[list(mono_keyframes)] = True
    obs_kf, obs_lm, obs_xy, obs_xr, inv_s, is_outlier = [], [], [], [], [], []
    for l, kfs in enumerate(view_sets):
        for k in kfs:
            uv, _ = synth.project(cam, poses[k], points[l])
            noise = rng.standard_normal(3) * pixel_sigma
            out = rng.random() < outlier_frac
            if out:
                noise[:2] += rng.choice([-1, 1], 2) * rng.uniform(15, 40, 2)
            obs_kf.append(k); obs_lm.append(l)
            obs_xy.append((uv[0] + noise[0], uv[1] + noise[1]))
            obs_xr.append(uv[2] + noise[2] if (stereo and not mono_kf[k] and not mono_lm[l]) else -1.0)
            inv_s.append(1.0 / (1.2 ** int(rng.integers(0, 8))) ** 2)
            is_outlier.append(out)
    poses0 = poses.copy()
    for k in free_ids:
        R = poses[k, :9].reshape(3, 3); t = poses[k, 9:]
        dR = synth._rot(pose_noise[0] * rng.standard_normal(3))
        poses0[k, :9] = (dR @ R).reshape(-1); poses0[k, 9:] = dR @ t + pose_noise[1] * rng.standard_normal(3)
    points0 = points + point_noise * rng.standard_normal(points.shape)
    if seam:
        # behind free keyframe j, 2-3.2 m away, observed just left of the longitude seam and estimated just right of it: the
        # residual is a whole image width, the undamped step swings the point around the camera, and the first iterations
        # reject trial after trial until the damping is large enough (6 trials at seed 1 with 4 free + 2 fixed keyframes)
        assert model == "equirectangular" and num_free >= 2
        new_xy, new_kf, new_lm = [], [], []
        for j in range(seam):
            k, k2 = int(free_ids[j % num_free]), int(free_ids[(j + 1) % num_free])
            d, y, eps = 2.0 * (1 + 0.3 * j), 0.1 * j, 0.02
            pc_true = d * np.array([np.sin(np.pi - eps), y, np.cos(np.pi - eps)])
            pc_est = d * np.array([np.sin(-np.pi + eps), y, np.cos(-np.pi + eps)])
            pw = poses[k, :9].reshape(3, 3).T @ (pc_true - poses[k, 9:])
            points = np.vstack([points, pw])
            points0 = np.vstack([points0, poses0[k, :9].reshape(3, 3).T @ (pc_est - poses0[k, 9:])])
            for kk in sorted((k, k2)):
                uv, _ = synth.project(cam, poses[kk], pw)
                obs_kf.append(kk); obs_lm.append(len(points) - 1); obs_xy.append((uv[0], uv[1])); obs_xr.append(-1.0)
                inv_s.append(1.0); is_outlier.append(False)
    g = dict(cam=cam, setup_is_mono=not stereo, poses_gt=poses, points_gt=points, poses=poses0, points=points0, fixed=fx,
             obs_kf=np.array(obs_kf, np.int32), obs_lm=np.array(obs_lm, np.int32), obs_xy=np.array(obs_xy, np.float32).reshape(-1, 2),
             obs_xr=np.array(obs_xr, np.float32), inv_sigma_sq=np.array(inv_s, np.float32), is_outlier=np.array(is_outlier, bool),
             free_ids=free_ids)
    g["reduced_dim"] = 6 * num_free
    g["co_observations"] = co_observations(g)
    return g


def pose_graph(n, stereo=False, bad=0, seed=0):
    """Motion-only problem: one free keyframe, n landmarks (constants: `points` are the true positions) seen once each, so that
    `points` doubles as the per-edge pts_w of pose_optimizer.  bad > 0: pixel noise 0.3, a start close to the truth, no random
    outliers; the first `bad` observations are moved by 60 px (in four directions, so that their pulls cancel) and weighted as
    the coarsest pyramid level, the others as level 0."""
    g = graph(1, 0, num_landmarks=n, views=(1, 1), stereo=stereo, seed=seed, point_noise=0.0, outlier_frac=0.0 if bad else 0.1,
              pixel_sigma=0.3 if bad else 1.0, pose_noise=(0.0005, 0.002) if bad else (0.01, 0.05))
    g["points"] = g["points_gt"].copy()
    if bad:
        sign = np.array([[1, 1], [-1, -1], [1, -1], [-1, 1]], np.float32)
        g["obs_xy"][:bad] += np.float32(60.0) * sign[np.arange(bad) % 4]
        g["inv_sigma_sq"][:] = 1.0
        g["inv_sigma_sq"][:bad] = np.float32(1.0 / 1.2 ** 14)
        g["is_outlier"][:bad] = True
    return g


def args(g):
    """(poses, fixed, points, obs_kf, obs_lm, obs_xy, obs_xr or None, inv_sigma_sq) as the optimisers take them"""
    return (g["poses"], g["fixed"], g["points"], g["obs_kf"], g["obs_lm"], g["obs_xy"], None if g["setup_is_mono"] else g["obs_xr"],
            g["inv_sigma_sq"])


def _free_edges_per_landmark(g):
    on_free = g["fixed"][g["obs_kf"]] == 0
    return np.bincount(g["obs_lm"][on_free], minlength=len(g["points"]))


def co_observations(g):
    """co-observation entries of the graph: m (m + 1) / 2 per landmark over its m edges on free keyframes (diagonal included)"""
    m = _free_edges_per_landmark(g).astype(np.int64)
    return int((m * (m + 1) // 2).sum())


def pair_co_observations(g, a, b):
    """landmarks seen by both free keyframes a and b (ordinals among the free keyframes)"""
    ka, kb = g["free_ids"][a], g["free_ids"][b]
    la = set(g["obs_lm"][g["obs_kf"] == ka].tolist()); lb = set(g["obs_lm"][g["obs_kf"] == kb].tolist())
    return len(la & lb)


# ----------------------------------------------------------------------------------------------------- float64 reference
def huber_delta(setup_is_mono):
    """g2o's Huber width: sqrt of the chi2 bound as the reference computes it (float sqrtf)"""
    return float(np.sqrt(np.float32(CHI2_2D if setup_is_mono else CHI2_3D)))


def _errors(g, poses, points, xr):
    """(M, 3) residuals obs - project, third column zero for monocular edges (numpy projection, no oracle code)"""
    M = len(g["obs_kf"])
    e = np.zeros((M, 3))
    for k in np.unique(g["obs_kf"]):
        idx = np.flatnonzero(g["obs_kf"] == k)
        uv, _ = synth.project(g["cam"], poses[k], points[g["obs_lm"][idx]])
        e[idx, 0] = g["obs_xy"][idx, 0].astype(np.float64) - uv[:, 0]
        e[idx, 1] = g["obs_xy"][idx, 1].astype(np.float64) - uv[:, 1]
        if xr is not None and g["cam"]["model"] != "equirectangular":
            st = xr[idx] >= 0
            e[idx[st], 2] = xr[idx][st].astype(np.float64) - uv[st, 2]
    return e


def _robust_chi2(g, poses, points, xr, active, delta):
    c = (_errors(g, poses, points, xr) ** 2).sum(1) * g["inv_sigma_sq"].astype(np.float64)
    c = c[active]
    if delta is None:
        return float(c.sum())
    d2 = delta * delta
    return float(np.where(c <= d2, c, 2 * np.sqrt(c) * delta - d2).sum())


def full_system(oracle, g, poses, points, xr, active, delta, with_points):
    """The full normal equations at the current state, linearised edge by edge through `oracle.edge_eval`: H (sparse,
    poses then points) and b = -J^T W e.  Returns the linear system as `reference_lm` takes it: diag (of H), b, free_idx and
    solve(lam) = (H + lam I)^-1 b by scipy's sparse LU."""
    cam = oracle.camera(**g["cam"])
    free_idx = np.cumsum(g["fixed"] == 0) - 1
    free_idx[g["fixed"] != 0] = -1
    nfree = int((g["fixed"] == 0).sum())
    n, L = 6 * nfree, len(points)
    N = n + (3 * L if with_points else 0)
    rows, cols, vals = [], [], []
    b = np.zeros(N)
    for i in np.flatnonzero(active):
        k, l = int(g["obs_kf"][i]), int(g["obs_lm"][i])
        stereo = xr is not None and xr[i] >= 0
        obs = np.array([g["obs_xy"][i, 0], g["obs_xy"][i, 1], xr[i] if xr is not None else -1.0], np.float64)
        e, Jp, Jl, _ = oracle.edge_eval(cam, poses[k], points[l], obs, stereo)
        w = float(g["inv_sigma_sq"][i])
        chi = w * float(e @ e)
        ww = w * (1.0 if delta is None or chi <= delta * delta else delta / np.sqrt(chi))
        blocks = []
        if free_idx[k] >= 0:
            blocks.append((6 * free_idx[k], Jp))
        if with_points:
            blocks.append((n + 3 * l, Jl))
        for oa, Ja in blocks:
            b[oa:oa + Ja.shape[1]] -= Ja.T @ (ww * e)
            for ob, Jb in blocks:
                blk = ww * (Ja.T @ Jb)
                r, c = np.meshgrid(np.arange(Ja.shape[1]) + oa, np.arange(Jb.shape[1]) + ob, indexing="ij")
                rows.append(r.ravel()); cols.append(c.ravel()); vals.append(blk.ravel())
    H = sp.coo_matrix((np.concatenate(vals) if vals else np.zeros(0), (np.concatenate(rows) if rows else np.zeros(0, int),
                      np.concatenate(cols) if cols else np.zeros(0, int))), shape=(N, N)).tocsc()
    return SimpleNamespace(diag=H.diagonal(), b=b, free_idx=free_idx,
                           solve=lambda lam: spla.spsolve((H + lam * sp.identity(N, format="csc")).tocsc(), b))


def reference_lm(oracle, g, iterations, use_huber=True, with_points=True, level=None, poses=None, points=None, system=None, oplus=None):
    """g2o's OptimizationAlgorithmLevenberg on the full normal equations.  Returns (poses, points, dict(lambda_init,
    trials = trials per iteration, states = [(poses, points)] after each iteration)).  `level` marks excluded edges;
    with_points=False keeps the points constant (motion-only problem).  `system(g, poses, points, xr, active, delta,
    with_points)` linearises (default: `full_system` through the oracle's edges) and `oplus(poses (k, 12), dx (k, 6))`
    updates the free poses (default: `oracle.pose_oplus`): the driver is shared with the vectorised reference of
    tests/ba_reference64.py."""
    if system is None:
        system = functools.partial(full_system, oracle)
    if oplus is None:
        oplus = lambda ps, us: np.array([oracle.pose_oplus(p, u) for p, u in zip(ps, us)]).reshape(-1, 12)
    poses = np.array(g["poses"] if poses is None else poses, np.float64).copy()
    points = np.array(g["points"] if points is None else points, np.float64).copy()
    xr = None if g["setup_is_mono"] else g["obs_xr"]
    active = np.ones(len(g["obs_kf"]), bool) if level is None else ~np.asarray(level, bool)
    delta = huber_delta(g["setup_is_mono"]) if use_huber else None
    lam, ni, lam0 = 0.0, 2.0, None
    trials, states = [], []
    cur = _robust_chi2(g, poses, points, xr, active, delta)
    for it in range(iterations):
        lin = system(g, poses, points, xr, active, delta, with_points)
        free = np.flatnonzero(lin.free_idx >= 0)
        n = 6 * len(free)
        if it == 0:
            lam = 1e-5 * float(np.abs(lin.diag).max())
            lam0, ni = lam, 2.0
        q = 0
        while True:
            dx = lin.solve(lam)
            cp = poses.copy()
            cp[free] = oplus(poses[free], dx[:n].reshape(-1, 6)[lin.free_idx[free]])
            cq = points + dx[n:].reshape(-1, 3) if with_points else points
            new = _robust_chi2(g, cp, cq, xr, active, delta)
            rho = (cur - new) / (float(dx @ (lam * dx + lin.b)) + 1e-3)
            q += 1
            if rho > 0 and np.isfinite(new):
                lam *= max(1.0 / 3.0, min(1.0 - (2 * rho - 1) ** 3, 2.0 / 3.0))
                ni = 2.0
                cur = new
                poses, points = cp, cq
            else:
                lam *= ni
                ni *= 2
            if not (rho < 0 and q < 10):
                break
        trials.append(q)
        states.append((poses.copy(), points.copy()))
        if q == 10 or rho == 0:
            break
    return poses, points, dict(lambda_init=lam0, trials=trials, states=states)


def step_error(x, x_ref, x_start):
    """||(x - x_start) - (x_ref - x_start)||_inf / ||x_ref - x_start||_inf: the error of a step relative to the step"""
    x, x_ref, x_start = (np.asarray(a, np.float64) for a in (x, x_ref, x_start))
    return float(np.abs(x - x_ref).max() / np.abs(x_ref - x_start).max())
