"""The optimisers' Levenberg STEPS on the GPU: one and two iterations through the public entry points, against the oracle and
(where the graph is small enough) against the float64 full-system reference of tests/ba_graphs.py.  A step is the solution of
the damped normal equations, so an error in the Schur complement, the reduced Cholesky or the back-substitution shows up in it
at its own size; the converged results that test_optimize_gpu.py compares cannot see such errors (a wrong Hessian only changes
the path to the same fixed point).  The graphs sit on the solver's size switches and on the degenerate parts that synthetic
maps never contain."""
import functools

import numpy as np
import pytest

import ba_graphs as bg

pytestmark = pytest.mark.gpu

# |(x_gpu - x_start) - (x_ref - x_start)|_inf / |x_ref - x_start|_inf, poses and points separately, after 1 and 2 iterations.
# Measured on an H100 SXM (80 GB), largest over every case below: GPU vs oracle 1.5e-13 (pose optimiser, n = 2049; 1.0e-13
# for the BA steps), GPU vs the float64 reference 7.7e-12 (points of free62: the reference factorises the full system by sparse
# LU, the damped system's conditioning amplifies the different rounding).  TOL is 13x above the largest.
MEASURED = 7.7e-12
TOL = 1e-10
REF_MAX_EDGES = 4000          # the python reference linearises edge by edge: only for the smaller graphs

C = {(5, 6): 127, (6, 7): 128, (7, 8): 129, (8, 0): 257}
LOCAL = {
    # reduced dimension n = 6, 12 (one narrow block), 96 (no narrow last block)
    "free1": dict(num_free=1, num_fixed=2, num_landmarks=150, seed=11),
    "free2": dict(num_free=2, num_fixed=2, num_landmarks=200, seed=12),
    "free16": dict(num_free=16, num_fixed=3, num_landmarks=500, seed=13),
    # double- / single-buffered back-substitution (n = 372 / 378); one / two radix-sort passes (2016 / 2080 pairs)
    "free62": dict(num_free=62, num_fixed=4, num_landmarks=900, views=(2, 6), seed=14),
    "free63": dict(num_free=63, num_fixed=4, num_landmarks=900, views=(2, 6), seed=15),
    "free64": dict(num_free=64, num_fixed=4, num_landmarks=900, views=(2, 6), seed=16),
    # cluster Cholesky (n = 684) / multi-launch k_chol_big_* (n = 690)
    "free114": dict(num_free=114, num_fixed=3, num_landmarks=1200, views=(2, 6), seed=17),
    "free115": dict(num_free=115, num_fixed=3, num_landmarks=1200, views=(2, 6), seed=18),
    # free index != keyframe id
    "keyframe0_fixed": dict(num_free=20, num_fixed=1, fixed="first", num_landmarks=500, seed=19),
    "every_third_fixed": dict(num_free=30, num_fixed=15, fixed="interleaved", num_landmarks=700, seed=20),
    # k_ba_free_index carries its prefix over tiles of 1024 keyframes
    "k1100_free150": dict(num_free=150, num_fixed=950, fixed="interleaved", num_landmarks=2500, views=(2, 6), seed=21),
    # Schur packing (four co-observations per three DMMAs) and chunk remainders (128 records per chunk)
    "pair_counts": dict(num_free=10, num_fixed=3, fixed="interleaved", num_landmarks=150, seed=22,
                        pair_counts={(0, 1): 1, (1, 2): 2, (2, 3): 3, (3, 4): 4, (4, 5): 5, **C}),
    # empty diagonal segments, lm_first gaps at both ends, rank-2 Hll, m (m + 1) / 2 emissions from one thread
    "degenerate": dict(num_free=12, num_fixed=4, fixed="interleaved", num_landmarks=300, empty_free=(0, 7), unobserved=6, fixed_only=5,
                       single_view=8, seen_by_all=2, seed=23),
    # 2- and 3-row edges in one system; negative depths for the classifier after round 1
    "stereo_mono_keyframes": dict(num_free=10, num_fixed=3, fixed="first", num_landmarks=400, stereo=True, mono_keyframes=(0, 4, 5, 9, 11),
                                  behind=6, seed=24),
    # the first iteration rejects five trials: the device halts after its batch of four, k_lm_resume + a second batch finish it
    "seam_rejections": dict(num_free=4, num_fixed=2, fixed="first", num_landmarks=60, model="equirectangular", seam=3, seed=1),
}
GLOBAL = ["free2", "free64", "k1100_free150", "degenerate", "seam_rejections"]


@functools.lru_cache(maxsize=None)
def _graph(name):
    return bg.graph(**LOCAL[name])


@functools.lru_cache(maxsize=None)
def _reference(name):
    from oracle import oracle as O
    O.build()
    g = _graph(name)
    if len(g["obs_kf"]) > REF_MAX_EDGES:
        return None
    return bg.reference_lm(O, g, 2)[2]


def run_ba(oracle, name, kind, it):
    """one optimiser call of `it` iterations on the GPU and in the oracle -> results and step-error ratios"""
    return run_ba_graph(oracle, _graph(name), _reference(name), kind, it)


def run_ba_graph(oracle, g, ref, kind, it):
    """run_ba on graph g, with the reference's Levenberg record `ref` (or None)"""
    from openvslam_b200 import optimize
    mono = g["setup_is_mono"]
    if kind == "local":
        ba = optimize.local_bundle_adjuster(it, 0)
        poses, points, outl, st = ba.optimize(optimize.camera(**g["cam"]), mono, *bg.args(g))
        oposes, opoints, ooutl, ost = oracle.local_ba(oracle.camera(**g["cam"]), mono, *bg.args(g), num_first_iter=it, num_second_iter=0)
    else:
        ba = optimize.global_bundle_adjuster(it, True)
        poses, points, st = ba.optimize(optimize.camera(**g["cam"]), mono, *bg.args(g))
        oposes, opoints, ost = oracle.global_ba(oracle.camera(**g["cam"]), mono, *bg.args(g), num_iter=it)
        outl = ooutl = None
    ba.close()
    r = dict(g=g, st=st, ost=ost, outl=outl, ooutl=ooutl, poses=poses,
             pose_vs_oracle=bg.step_error(poses, oposes, g["poses"]), point_vs_oracle=bg.step_error(points, opoints, g["points"]))
    if ref is not None:
        rp, rq = ref["states"][it - 1]
        assert sum(ref["trials"][:it]) == ost["num_trials"]
        r.update(pose_vs_ref=bg.step_error(poses, rp, g["poses"]), point_vs_ref=bg.step_error(points, rq, g["points"]))
    return r


def _check(r):
    g, st, ost = r["g"], r["st"], r["ost"]
    assert st["reduced_dim"] == g["reduced_dim"] and st["co_observations"] == g["co_observations"]
    assert st["lambda_init"][0] == pytest.approx(ost["lambda_init"][0], rel=1e-10)
    assert st["num_trials"] == ost["num_trials"] and st["num_iterations"] == ost["num_iterations"]
    assert np.array_equal(r["poses"][g["fixed"] == 1], g["poses"][g["fixed"] == 1])
    for key in ("pose_vs_oracle", "point_vs_oracle", "pose_vs_ref", "point_vs_ref"):
        if key in r:
            assert r[key] <= TOL, (key, r[key])
    if r["outl"] is not None:
        assert np.array_equal(r["outl"], r["ooutl"])


@pytest.mark.parametrize("it", [1, 2])
@pytest.mark.parametrize("name", list(LOCAL))
def test_local_ba_steps(oracle, name, it):
    r = run_ba(oracle, name, "local", it)
    _check(r)
    if name == "seam_rejections" and it == 1:
        assert r["ost"]["num_trials"] >= 5                     # beyond the first speculative batch of four
    if name == "stereo_mono_keyframes":
        assert r["outl"].sum() >= 12                            # the 6 x 2 edges behind the cameras, cut by the depth test


@pytest.mark.parametrize("it", [1, 2])
@pytest.mark.parametrize("name", GLOBAL)
def test_global_ba_steps(oracle, name, it):
    _check(run_ba(oracle, name, "global", it))


def run_pose(oracle, n, stereo, bad=0, num_trials=1):
    return run_pose_graph(oracle, bg.pose_graph(n, stereo=stereo, bad=bad, seed=n), num_trials)


def run_pose_graph(oracle, g, num_trials=1, ref=None):
    """pose_optimizer(num_trials, 1) on the GPU and in the oracle on the motion-only graph g (edge i sees g["points"][i]), and
    one reference iteration (`ref`: its Levenberg record, computed here when None)"""
    from openvslam_b200 import optimize
    xr = None if g["setup_is_mono"] else g["obs_xr"]
    args = (g["setup_is_mono"], g["points"], g["obs_xy"], xr, g["inv_sigma_sq"], g["poses"][0])
    po = optimize.pose_optimizer(num_trials, 1)
    ninl, pose, flags, st = po.optimize(optimize.camera(**g["cam"]), *args)
    po.close()
    on, opose, oflags, ost = oracle.pose_optimize(oracle.camera(**g["cam"]), *args, num_trials=num_trials, num_each_iter=1)
    info = bg.reference_lm(oracle, g, 1, with_points=False)[2] if ref is None else ref
    rp = info["states"][0][0]
    return dict(ninl=ninl, on=on, flags=flags, oflags=oflags, st=st, ost=ost, ref_trials=info["trials"], ref_lambda_init=info["lambda_init"],
                pose_vs_oracle=bg.step_error(pose, opose, g["poses"][0]), pose_vs_ref=bg.step_error(pose, rp[0], g["poses"][0]))


@pytest.mark.parametrize("n,stereo", [(5, True), (2047, False), (2048, True), (2049, False), (4097, True)])
def test_pose_optimizer_step(oracle, n, stereo):
    """one round of one iteration around the 8 x 256-thread cluster stride of k_pose_optimize"""
    r = run_pose(oracle, n, stereo)
    assert r["ninl"] == r["on"] and np.array_equal(r["flags"], r["oflags"])
    assert r["st"]["lambda_init"][0] == pytest.approx(r["ost"]["lambda_init"][0], rel=1e-10)
    assert r["st"]["num_trials"] == r["ost"]["num_trials"] == r["ref_trials"][0]
    assert r["pose_vs_oracle"] <= TOL and r["pose_vs_ref"] <= TOL


def test_pose_optimizer_stops_below_five_inliers(oracle):
    """four of eight edges are outliers after round 1: n - num_bad < 5 ends the call after that round"""
    r = run_pose(oracle, 8, False, bad=4, num_trials=4)
    assert r["ninl"] == r["on"] == 4 and np.array_equal(r["flags"], r["oflags"]) and r["flags"][:4].all()
    assert r["st"]["num_rounds"] == r["ost"]["num_rounds"] == 1
    assert r["pose_vs_oracle"] <= TOL and r["pose_vs_ref"] <= TOL
