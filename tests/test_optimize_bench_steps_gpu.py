"""The optimisers' Levenberg STEPS at the benchmark's problem shapes: the local BA of bench.py's configs 4 and 5 (50 free + 10
fixed keyframes, 20 000 landmarks, ~100 000 edges), the global BA on config 4's graph and the pose optimiser on the pose
problems of configs 2-5, each against the oracle and against the vectorised float64 reference of tests/ba_reference64.py.
At this size every free keyframe's diagonal pair holds 13-14 chunks of 128 co-observation records (the in-order chunk sums
of k_ba_schur_final and k_ba_pose_accum_chunk) and the 1275 keyframe pairs take two 1024-pair tiles of k_ba_chunk_scan;
the converged comparisons of test_optimize_gpu.py cannot see an error there.  Smaller graphs isolate one feature each: an
off-diagonal pair of many chunks, a keyframe of more than 32 chunks, and more than 1024 pairs.

The problems are built the way bench.make_workload builds rank 0's, from bench's own constants, so that a change of the
benchmark's workload moves these tests with it.  The oracle's steps at the same shapes agree with the reference to 2e-13
(test_ba_reference64.py); a GPU error far above that is a kernel bug, not the conditioning of the damped system."""
import functools

import numpy as np
import pytest

import ba_graphs as bg
import ba_reference64 as R
from test_optimize_steps_gpu import TOL, _check, run_ba_graph, run_pose_graph

pytestmark = pytest.mark.gpu

BA_CONFIGS = [c for c, cfg in R.bench_module().CONFIGS.items() if cfg["ba"]]
POSE_CONFIGS = sorted(R.bench_module().CONFIGS)

SYNTH = {
    # off-diagonal pairs of 383 / 384 / 385 records: three chunks, three full chunks, a fourth of one record
    "pairs_383_384_385": dict(num_free=8, num_fixed=2, fixed="interleaved", num_landmarks=200, seed=31,
                              pair_counts={(0, 1): 383, (2, 3): 384, (4, 5): 385}),
    # off-diagonal pairs of 8 and 33 chunks
    "pairs_1000_4097": dict(num_free=6, num_fixed=2, num_landmarks=150, seed=32, pair_counts={(0, 1): 1000, (2, 3): 4097}),
    # free keyframe 0 has > 4096 edges (> 32 chunks of k_ba_pose_accum_chunk), every off-diagonal pair at most three chunks
    "keyframe_4200_edges": dict(num_free=14, num_fixed=2, num_landmarks=200, seed=33, pair_counts={(0, b): 350 for b in range(1, 13)}),
    # 46 fully co-visible free keyframes: 1081 pairs, past the first 1024-pair tile of k_ba_chunk_scan
    "covisible46_equirectangular": dict(num_free=46, num_fixed=2, num_landmarks=200, seen_by_all=30, model="equirectangular", seed=34),
}


@functools.lru_cache(maxsize=None)
def _synth(name):
    g = bg.graph(**SYNTH[name])
    return g, R.reference_lm(g, 2)[2]


def _check_ref(r, ref):
    assert r["st"]["lambda_init"][0] == pytest.approx(ref["lambda_init"], rel=1e-10)
    assert r["pose_vs_ref"] <= TOL and r["point_vs_ref"] <= TOL, (r["pose_vs_ref"], r["point_vs_ref"])


def _report(label, r):
    print("%s: GPU vs oracle pose %.1e point %.1e, GPU vs reference pose %.1e point %.1e"
          % (label, r["pose_vs_oracle"], r["point_vs_oracle"], r["pose_vs_ref"], r["point_vs_ref"]))


@pytest.mark.parametrize("it", [1, 2])
@pytest.mark.parametrize("config", BA_CONFIGS)
def test_local_ba_steps_at_benchmark_shape(oracle, config, it):
    g = R.bench_ba_problem(config)
    npairs, diag_chunks, _ = R.pair_chunks(g)
    assert npairs > 1024 and diag_chunks >= 13          # two scan tiles; >= 13 chunks on every diagonal pair
    ref = R.bench_ba_reference(config)
    r = run_ba_graph(oracle, g, ref, "local", it)
    _report("config %d local BA, %d iteration(s)" % (config, it), r)
    assert r["st"]["reduced_dim"] == 300
    _check(r)
    _check_ref(r, ref)


@pytest.mark.parametrize("it", [1, 2])
def test_global_ba_steps_at_benchmark_shape(oracle, it):
    g = R.bench_ba_problem(4)
    ref = R.bench_ba_reference(4)
    r = run_ba_graph(oracle, g, ref, "global", it)
    _report("config 4 global BA, %d iteration(s)" % it, r)
    _check(r)
    _check_ref(r, ref)


def test_synthetic_graphs_have_their_shapes():
    g, _ = _synth("pairs_383_384_385")
    assert [bg.pair_co_observations(g, a, a + 1) for a in (0, 2, 4)] == [383, 384, 385]
    g, _ = _synth("pairs_1000_4097")
    assert bg.pair_co_observations(g, 0, 1) == 1000 and bg.pair_co_observations(g, 2, 3) == 4097
    g, _ = _synth("keyframe_4200_edges")
    assert (g["obs_kf"] == g["free_ids"][0]).sum() > 4096 and R.pair_chunks(g)[2] <= 384
    g, _ = _synth("covisible46_equirectangular")
    assert R.pair_chunks(g)[0] == 46 * 47 // 2


@pytest.mark.parametrize("it", [1, 2])
@pytest.mark.parametrize("name", list(SYNTH))
def test_local_ba_steps_on_chunk_graphs(oracle, name, it):
    g, ref = _synth(name)
    r = run_ba_graph(oracle, g, ref, "local", it)
    _report("%s local BA, %d iteration(s)" % (name, it), r)
    _check(r)
    _check_ref(r, ref)


@pytest.mark.parametrize("config", POSE_CONFIGS)
def test_pose_optimizer_step_at_benchmark_shape(oracle, config):
    """one round of one iteration on the benchmark's pose problem: 1000 / 2000 stereo / 4000 equirectangular / 2000 edges"""
    g = R.bench_pose_problem(config)
    ref = R.bench_pose_reference(config)
    r = run_pose_graph(oracle, g, 1, ref)
    print("config %d pose optimiser: GPU vs oracle %.1e, GPU vs reference %.1e" % (config, r["pose_vs_oracle"], r["pose_vs_ref"]))
    assert r["ninl"] == r["on"] and np.array_equal(r["flags"], r["oflags"])
    assert r["st"]["lambda_init"][0] == pytest.approx(r["ost"]["lambda_init"][0], rel=1e-10)
    assert r["st"]["lambda_init"][0] == pytest.approx(r["ref_lambda_init"], rel=1e-10)
    assert r["st"]["num_trials"] == r["ost"]["num_trials"] == r["ref_trials"][0]
    assert r["pose_vs_oracle"] <= TOL and r["pose_vs_ref"] <= TOL
