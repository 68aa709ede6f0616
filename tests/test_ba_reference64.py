"""The vectorised float64 reference of tests/ba_reference64.py, pinned before anything is compared with it: its edges against
the oracle's and against finite differences, its Levenberg steps against the full-system reference of tests/ba_graphs.py, its
point-eliminated solve against one sparse LU of the whole system; and, at the benchmark's two local-BA shapes, the oracle's
steps against it -- the yardstick the GPU's errors in test_optimize_bench_steps_gpu.py are read against."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import ba_graphs as bg
import ba_reference64 as R
from test_optimize_steps_gpu import LOCAL, REF_MAX_EDGES, TOL, _graph

# vectorised vs full-system reference after one or two iterations: the same damped system solved two ways (point
# elimination + dense Cholesky, sparse LU of the whole system).  Measured <= 7.7e-12 of the step (points of free62; <= 3.4e-12
# on every other graph): the conditioning of the damped system, not a different system.
LM_TOL = 2e-11
POSE_GRAPHS = [(5, True), (300, True), (2047, False), (2048, True), (4097, True)]
BENCH_POSE = [2, 3, 4, 5]


EDGE_CASES = list(LOCAL) + ["pose%d_%s" % (n, "stereo" if st else "mono") for n, st in POSE_GRAPHS] + ["bench_pose%d" % c for c in BENCH_POSE]


def _edge_graph(name):
    if name in LOCAL:
        return _graph(name)
    if name.startswith("bench_pose"):
        return R.bench_pose_problem(int(name[len("bench_pose"):]))
    n, kind = name[len("pose"):].split("_")
    return bg.pose_graph(int(n), stereo=kind == "stereo", seed=int(n))


def _xr(g):
    return None if g["setup_is_mono"] else g["obs_xr"]


@pytest.mark.parametrize("name", EDGE_CASES)
def test_edges_equal_oracle(oracle, name):
    """residuals and both Jacobians of every edge equal oracle.edge_eval's to ~1e-15 relative (the same formulas, restated)"""
    g = _edge_graph(name)
    xr = _xr(g)
    M = len(g["obs_kf"])
    e, Jp, Jl = R.edges(g, g["poses"], g["points"], xr, np.arange(M))
    cam = oracle.camera(**g["cam"])
    stereo_rows = 0
    for i in range(M):
        stereo = xr is not None and bool(xr[i] >= 0)
        obs = np.array([g["obs_xy"][i, 0], g["obs_xy"][i, 1], xr[i] if xr is not None else -1.0])
        eo, Jpo, Jlo, _ = oracle.edge_eval(cam, g["poses"][g["obs_kf"][i]], g["points"][g["obs_lm"][i]], obs, stereo)
        d = len(eo)
        stereo_rows += d == 3
        assert np.abs(e[i, :d] - eo).max() <= 1e-12 * np.abs(obs[:d]).max(), i
        assert np.abs(Jp[i, :d] - Jpo).max() <= 1e-12 * np.abs(Jpo).max(), i
        assert np.abs(Jl[i, :d] - Jlo).max() <= 1e-12 * np.abs(Jlo).max(), i
        assert not e[i, d:].any() and not Jp[i, d:].any() and not Jl[i, d:].any()
    assert (stereo_rows > 0) == (xr is not None)


@pytest.mark.parametrize("name", ["free16", "stereo_mono_keyframes", "seam_rejections", "bench_pose4"])
def test_jacobians_equal_finite_differences(name):
    """central differences of the residual under the pose update (pose_oplus) and a point move, independent of both
    restatements of the Jacobians"""
    g = _edge_graph(name)
    xr = _xr(g)
    M = min(len(g["obs_kf"]), 400)
    poses, pw = g["poses"][g["obs_kf"][:M]], g["points"][g["obs_lm"][:M]]
    obs = np.zeros((M, 3)); obs[:, :2] = g["obs_xy"][:M]
    stereo = np.zeros(M, bool) if xr is None else xr[:M] >= 0
    if xr is not None:
        obs[:, 2] = xr[:M]
    _, Jp, Jl = R.edge_eval(g["cam"], poses, pw, obs, stereo)
    h = 1e-6
    for j in range(6):
        u = np.zeros((M, 6)); u[:, j] = h
        fd = (R.edge_eval(g["cam"], R.pose_oplus(poses, u), pw, obs, stereo)[0] - R.edge_eval(g["cam"], R.pose_oplus(poses, -u), pw, obs, stereo)[0]) / (2 * h)
        assert np.abs(fd - Jp[:, :, j]).max() <= 1e-6 * np.abs(Jp).max(), j
    for j in range(3):
        d = np.zeros(3); d[j] = h
        fd = (R.edge_eval(g["cam"], poses, pw + d, obs, stereo)[0] - R.edge_eval(g["cam"], poses, pw - d, obs, stereo)[0]) / (2 * h)
        assert np.abs(fd - Jl[:, :, j]).max() <= 1e-6 * np.abs(Jl).max(), j
    assert np.allclose(R.se3_exp(np.zeros((1, 6)))[0], np.eye(3))


@pytest.mark.parametrize("name", [n for n in LOCAL if len(_graph(n)["obs_kf"]) <= REF_MAX_EDGES])
def test_lm_equals_full_system_reference(oracle, name):
    """ba_graphs.reference_lm on the vectorised edges and the point-eliminated solve = on the oracle's edges and a sparse LU
    of the full system: the same lambda_0, trial counts and (within the conditioning) states"""
    g = _graph(name)
    a = bg.reference_lm(oracle, g, 2)[2]
    b = R.reference_lm(g, 2)[2]
    assert b["lambda_init"] == pytest.approx(a["lambda_init"], rel=1e-12)
    assert b["trials"] == a["trials"]
    for (pa, qa), (pb, qb) in zip(a["states"], b["states"]):
        assert bg.step_error(pb, pa, g["poses"]) <= LM_TOL and bg.step_error(qb, qa, g["points"]) <= LM_TOL


@pytest.mark.parametrize("n,stereo", POSE_GRAPHS[:3])
def test_pose_lm_equals_full_system_reference(oracle, n, stereo):
    g = bg.pose_graph(n, stereo=stereo, seed=n)
    a = bg.reference_lm(oracle, g, 1, with_points=False)[2]
    b = R.reference_lm(g, 1, with_points=False)[2]
    assert b["lambda_init"] == pytest.approx(a["lambda_init"], rel=1e-12) and b["trials"] == a["trials"]
    assert bg.step_error(b["states"][0][0][0], a["states"][0][0][0], g["poses"][0]) <= 1e-12


def _solve_vs_lu(g, lam_factors=(1.0,)):
    lin = R.linearise(g, g["poses"], g["points"], _xr(g), np.ones(len(g["obs_kf"]), bool), bg.huber_delta(g["setup_is_mono"]), True)
    n = 6 * int((lin.free_idx >= 0).sum())
    worst = 0.0
    for f in lam_factors:
        lam = f * 1e-5 * np.abs(lin.diag).max()
        x, y = lin.solve(lam), spla.spsolve(lin.full(lam), lin.b)
        assert np.abs(lin.full(lam) @ y - lin.b).max() <= 1e-9 * np.abs(lin.b).max()
        worst = max(worst, np.abs(x[:n] - y[:n]).max() / np.abs(y[:n]).max(), np.abs(x[n:] - y[n:]).max() / np.abs(y[n:]).max())
    return worst


@pytest.mark.parametrize("name", ["free2", "free62", "pair_counts", "degenerate", "stereo_mono_keyframes", "seam_rejections"])
def test_point_elimination_equals_full_lu(name):
    assert _solve_vs_lu(_graph(name), (1.0, 64.0, 2.0 ** 15)) <= LM_TOL


def test_point_elimination_equals_full_lu_at_benchmark_shape():
    """once at config 4's 100 000 edges (the sparse LU alone takes ~30 s)"""
    assert _solve_vs_lu(R.bench_ba_problem(4)) <= LM_TOL


# -------------------------------------------------------------------------------------- the yardstick, before any GPU
@pytest.mark.parametrize("config", [4, 5])
def test_oracle_steps_at_benchmark_shape(oracle, config, capsys):
    """The oracle's 1- and 2-iteration local BA (and global BA) on the benchmark's problem against the reference: what two
    float64 solvers of the same damped system disagree by at this size, so that a GPU error far above it is a bug"""
    g = R.bench_ba_problem(config)
    ref = R.bench_ba_reference(config)
    cam = oracle.camera(**g["cam"])
    for it in (1, 2):
        op, oq, _, ost = oracle.local_ba(cam, True, *bg.args(g), num_first_iter=it, num_second_iter=0)
        gp, gq, gst = oracle.global_ba(cam, True, *bg.args(g), num_iter=it)
        rp, rq = ref["states"][it - 1]
        assert ost["lambda_init"][0] == pytest.approx(ref["lambda_init"], rel=1e-12)
        assert ost["num_trials"] == gst["num_trials"] == sum(ref["trials"][:it])
        errs = dict(local_pose=bg.step_error(op, rp, g["poses"]), local_point=bg.step_error(oq, rq, g["points"]),
                    global_pose=bg.step_error(gp, rp, g["poses"]), global_point=bg.step_error(gq, rq, g["points"]))
        with capsys.disabled():
            print("\nconfig %d, %d iteration(s), oracle vs reference: %s" % (config, it, ", ".join("%s %.1e" % kv for kv in errs.items())))
        assert max(errs.values()) <= TOL, errs


@pytest.mark.parametrize("config", BENCH_POSE)
def test_oracle_pose_step_at_benchmark_shape(oracle, config):
    g = R.bench_pose_problem(config)
    ref = R.bench_pose_reference(config)
    ninl, pose, flags, st = oracle.pose_optimize(oracle.camera(**g["cam"]), g["setup_is_mono"], g["pts_w"], g["obs_xy"], _xr(g),
                                                 g["inv_sigma_sq"], g["poses"][0], num_trials=1, num_each_iter=1)
    assert st["lambda_init"][0] == pytest.approx(ref["lambda_init"], rel=1e-12) and st["num_trials"] == ref["trials"][0]
    assert bg.step_error(pose, ref["states"][0][0][0], g["poses"][0]) <= TOL


def test_benchmark_graphs_reach_the_chunked_paths():
    """what makes the benchmark's local BA worth a step test of its own: more than one 1024-pair tile of k_ba_chunk_scan and
    at least 13 chunks of 128 records on every diagonal pair"""
    for config in (4, 5):
        npairs, diag_chunks, off_max = R.pair_chunks(R.bench_ba_problem(config))
        assert npairs > 1024 and diag_chunks >= 13 and off_max <= 384
