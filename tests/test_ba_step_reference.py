"""The BA oracle's Levenberg STEPS against a float64 reference that shares no linear algebra with it (tests/ba_graphs.py: the full
normal equations over poses and points, scipy's sparse LU, no Schur complement), one and two iterations at a time, on
irregular graphs; and the graph builder's graphs against the structure their parameters claim.  With the oracle's steps pinned
here, the GPU tests (test_optimize_steps_gpu.py) can hold the kernels to the oracle on graphs too large for the reference."""
import numpy as np
import pytest

import ba_graphs as bg

# oracle vs reference after one or two iterations: measured <= 9.4e-13 of the step (summation order and the two factorisations
# of the same damped system); 1e-10 leaves room and still sees any wrong block, weight or damping term
TOL = 1e-10

CASES = {
    "keyframe0_fixed": dict(num_free=4, num_fixed=1, fixed="first", num_landmarks=60, seed=1),
    "every_third_fixed": dict(num_free=6, num_fixed=3, fixed="interleaved", num_landmarks=60, seed=2),
    "pairs_1_2_3_5": dict(num_free=6, num_fixed=2, fixed="last", num_landmarks=40, pair_counts={(0, 1): 1, (1, 2): 2, (2, 3): 3, (4, 5): 5}, seed=3),
    "degenerate_parts": dict(num_free=5, num_fixed=3, fixed="interleaved", num_landmarks=40, empty_free=(2,), unobserved=4, fixed_only=3,
                             single_view=4, seen_by_all=2, seed=4),
    "stereo_mono_keyframes_behind": dict(num_free=5, num_fixed=2, fixed="first", num_landmarks=50, stereo=True, mono_keyframes=(0, 3, 4),
                                         behind=3, single_view=2, seed=5),
    "equirectangular": dict(num_free=4, num_fixed=2, fixed="interleaved", num_landmarks=50, model="equirectangular", seed=6),
}


def _cam(oracle, g):
    return oracle.camera(**g["cam"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_equals_oracle_steps(oracle, name):
    g = bg.graph(**CASES[name])
    rp, rq, info = bg.reference_lm(oracle, g, 2)
    for it in (1, 2):
        op, oq, _, ost = oracle.local_ba(_cam(oracle, g), g["setup_is_mono"], *bg.args(g), num_first_iter=it, num_second_iter=0)
        gp, gq, gst = oracle.global_ba(_cam(oracle, g), g["setup_is_mono"], *bg.args(g), num_iter=it)
        assert ost["lambda_init"][0] == pytest.approx(info["lambda_init"], rel=1e-12) and gst["lambda_init"][0] == ost["lambda_init"][0]
        assert ost["num_trials"] == gst["num_trials"] == sum(info["trials"][:it])
        sp, sq = info["states"][it - 1]
        for p, q in ((op, oq), (gp, gq)):
            assert bg.step_error(p, sp, g["poses"]) <= TOL and bg.step_error(q, sq, g["points"]) <= TOL
        assert np.array_equal(op[g["fixed"] == 1], g["poses"][g["fixed"] == 1])


def test_reference_follows_rejected_trials(oracle):
    """Landmarks estimated across the equirectangular seam: the first iteration rejects five trials (lambda_0 * 2^15 is
    accepted), more than one speculative batch of four -- the reference walks the same damping values."""
    g = bg.graph(4, 2, fixed="first", num_landmarks=60, model="equirectangular", seam=3, seed=1)
    rp, rq, info = bg.reference_lm(oracle, g, 2)
    op, oq, _, ost = oracle.local_ba(_cam(oracle, g), True, *bg.args(g), num_first_iter=1, num_second_iter=0)
    assert ost["num_trials"] == info["trials"][0] == 6
    assert bg.step_error(op, info["states"][0][0], g["poses"]) <= TOL and bg.step_error(oq, info["states"][0][1], g["points"]) <= TOL
    op, oq, _, ost = oracle.local_ba(_cam(oracle, g), True, *bg.args(g), num_first_iter=2, num_second_iter=0)
    assert ost["num_trials"] == sum(info["trials"])
    assert bg.step_error(op, info["states"][1][0], g["poses"]) <= TOL and bg.step_error(oq, info["states"][1][1], g["points"]) <= TOL


@pytest.mark.parametrize("n,stereo", [(5, True), (40, False), (300, True)])
def test_reference_equals_pose_optimizer_step(oracle, n, stereo):
    """pose_optimizer with one round of one iteration = one damped 6 x 6 Gauss-Newton step of the Huber cost"""
    g = bg.pose_graph(n, stereo=stereo, seed=n)
    rp, _, info = bg.reference_lm(oracle, g, 1, with_points=False)
    xr = None if g["setup_is_mono"] else g["obs_xr"]
    ninl, pose, flags, st = oracle.pose_optimize(_cam(oracle, g), g["setup_is_mono"], g["points"], g["obs_xy"], xr, g["inv_sigma_sq"], g["poses"][0],
                                                 num_trials=1, num_each_iter=1)
    assert st["lambda_init"][0] == pytest.approx(info["lambda_init"], rel=1e-12) and st["num_trials"] == info["trials"][0]
    assert bg.step_error(pose, rp[0], g["poses"][0]) <= TOL


def test_pose_optimizer_stops_when_fewer_than_five_inliers_remain(oracle):
    """four of eight edges are outliers after round 1: n - num_bad < 5 ends the call after that round's one step"""
    g = bg.pose_graph(8, bad=4, seed=7)
    rp, _, info = bg.reference_lm(oracle, g, 1, with_points=False)
    ninl, pose, flags, st = oracle.pose_optimize(_cam(oracle, g), True, g["points"], g["obs_xy"], None, g["inv_sigma_sq"], g["poses"][0],
                                                 num_trials=4, num_each_iter=1)
    assert ninl == 4 and st["num_rounds"] == 1 and flags.sum() == 4 and flags[:4].all()
    assert bg.step_error(pose, rp[0], g["poses"][0]) <= TOL


# ----------------------------------------------------------------------------------------------------- the builder itself
def test_builder_layout_and_fixed_patterns():
    for pattern, want in (("first", [0, 1]), ("last", [4, 5]), ("interleaved", [0, 3])):
        g = bg.graph(4, 2, fixed=pattern, num_landmarks=30, seed=1)
        assert np.flatnonzero(g["fixed"]).tolist() == want
        assert g["free_ids"].tolist() == np.flatnonzero(g["fixed"] == 0).tolist()
        assert np.all(np.diff(g["obs_lm"]) >= 0)                                    # grouped by landmark
        pairs = g["obs_kf"].astype(np.int64) * len(g["points"]) + g["obs_lm"]
        assert len(np.unique(pairs)) == len(pairs)                                  # no duplicate observation
        assert g["obs_xy"].shape == (len(g["obs_kf"]), 2) and g["reduced_dim"] == 24
    assert np.flatnonzero(bg.fixed_mask(30, 15, "interleaved")).tolist() == list(range(0, 45, 3))
    f = bg.fixed_mask(150, 950, "interleaved")
    assert (np.flatnonzero(f == 0) >= 1024).any() and (np.flatnonzero(f == 0) < 1024).any()


def test_builder_pair_counts_are_exact():
    counts = {(0, 1): 1, (1, 2): 2, (2, 3): 3, (3, 4): 4, (4, 5): 5, (5, 6): 127, (6, 7): 128, (7, 8): 129, (8, 0): 257}
    g = bg.graph(10, 3, fixed="interleaved", num_landmarks=150, pair_counts=counts, seed=2)
    for (a, b), c in counts.items():
        assert bg.pair_co_observations(g, a, b) == c
    assert bg.pair_co_observations(g, 0, 2) == 0                                    # named keyframes only meet through their pairs
    m = np.bincount(g["obs_lm"][g["fixed"][g["obs_kf"]] == 0], minlength=len(g["points"]))
    assert g["co_observations"] == int((m * (m + 1) // 2).sum())


def test_builder_degenerate_parts():
    g = bg.graph(6, 3, fixed="interleaved", num_landmarks=40, empty_free=(1, 4), unobserved=5, fixed_only=3, single_view=4, seen_by_all=2,
                 behind=3, stereo=True, mono_keyframes=(0,), seed=3)
    L, K = len(g["points"]), len(g["poses"])
    assert L == 40 + 5 + 3 + 4 + 2 + 3
    per_lm = np.bincount(g["obs_lm"], minlength=L)
    assert per_lm[0] == 0 and per_lm[-1] == 0 and (per_lm == 0).sum() == 5         # unobserved: first, last and three more
    per_kf = np.bincount(g["obs_kf"], minlength=K)
    assert per_kf[g["free_ids"][1]] == 0 and per_kf[g["free_ids"][4]] == 0 and (per_kf[g["free_ids"][[0, 2, 3, 5]]] > 0).all()
    on_fixed = g["fixed"][g["obs_kf"]] == 1
    only_fixed = [l for l in range(L) if per_lm[l] and on_fixed[g["obs_lm"] == l].all()]
    assert len(only_fixed) >= 3
    single = [l for l in range(L) if per_lm[l] == 1]
    assert len(single) >= 4 and all(g["obs_xr"][g["obs_lm"] == l][0] < 0 for l in single)   # single views are monocular
    assert (per_lm == 4).sum() >= 2                                                  # seen by all four non-empty free keyframes
    assert (g["obs_xr"][g["obs_kf"] == 0] < 0).all() and (g["obs_xr"] >= 0).any()
    depth = np.einsum("mj,mj->m", g["poses_gt"][g["obs_kf"], 6:9], g["points_gt"][g["obs_lm"]]) + g["poses_gt"][g["obs_kf"], 11]
    assert (depth < 0).sum() == 6 and (depth[depth > 0] > 3).all()                  # 3 landmarks x 2 views behind the cameras
