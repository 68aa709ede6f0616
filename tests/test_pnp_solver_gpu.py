"""solve::pnp_solver on the GPU (k_pnp_hypotheses + k_pnp_ransac + k_pnp_refine: three launches per batch) against the oracle
(oracle/pnp_solver_oracle.c) and ground truth.  The kernels give every hypothesis one thread for EPnP and then a warp whose lanes
take the correspondences with a stride of 32, put 4 hypotheses in a CTA, and recompute with one 256-thread CTA per problem whose
sums take 256 strided partials; the sizes below sit around those strides."""
import os
import subprocess
import types

import numpy as np
import pytest

import pnp_problems as pp

pytestmark = pytest.mark.gpu

SIZES = [6, 7, 31, 32, 33, 255, 256, 257, 1000, 4000]
IDENTITY = np.concatenate([np.eye(3).ravel(), [0, 0, 0]])


@pytest.fixture(scope="module")
def ps(oracle):
    """the solver's oracle (oracle/pnp_solver.py); `oracle` builds liboracle.so"""
    from oracle import pnp_solver
    return pnp_solver


def _oracle(ps, p, min_num_inliers, max_num_iter, recompute, seed):
    return ps.pnp_solve_ransac(*pp.args(p), min_num_inliers=min_num_inliers, max_num_iter=max_num_iter, recompute=recompute, seed=seed)


def _same(g, o):
    assert g["valid"] == o["valid"]
    assert g["num_inliers"] == o["num_inliers"] and g["best_iter"] == o["best_iter"]
    assert np.array_equal(g["inliers"], o["inliers"])
    assert np.array_equal(g["pose_cw"], o["pose_cw"], equal_nan=True)


def _solve(problems, min_num_inliers=10, max_num_iter=30, recompute=True, seeds=None):
    from openvslam_b200 import solve
    s = solve.pnp_solver(min_num_inliers)
    out = s.find_via_ransac([pp.gpu_problem(p) for p in problems], max_num_iter, recompute, seeds)
    s.close()
    return out


@pytest.mark.parametrize("recompute", [True, False])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
def test_equals_oracle(ps, model, n, recompute):
    wrong = 0.1 + 0.3 * ((7 * n) % 10) / 10.0 if n > 7 else 0.0
    noise = 0.0 if n % 2 == 0 else 1e-3
    p = pp.problem(n, model=model, wrong=wrong, noise=noise, seed=n)
    min_inl = max(1, min(10, n // 2))
    g = _solve([p], min_inl, 30, recompute, [1000 + n])[0]
    o = _oracle(ps, p, min_inl, 30, recompute, 1000 + n)
    _same(g, o)
    if noise == 0.0:
        assert g["valid"] and np.abs(g["pose_cw"] - p["pose_true"]).max() <= 1e-9


@pytest.mark.parametrize("max_num_iter", [1, 3, 4, 5, 30, 31, 201])
def test_hypothesis_block_boundaries(ps, max_num_iter):
    p = pp.problem(300, wrong=0.4, noise=1e-3, seed=31)
    for recompute in (True, False):
        g = _solve([p], 10, max_num_iter, recompute, [5])[0]
        _same(g, _oracle(ps, p, 10, max_num_iter, recompute, 5))


def _mixed():
    """no correspondence, 5, fewer than min_num_inliers (10), coincident / collinear / planar sets, both bearing types, noisy
    and exact, 10-40 % wrong"""
    ps_ = [pp.problem(0, seed=1), pp.problem(5, wrong=0.0, seed=2), pp.problem(9, wrong=0.0, seed=3),
           pp.degenerate("coincident", seed=4), pp.degenerate("collinear", seed=5), pp.degenerate("planar", seed=6),
           pp.problem(300, model="equirectangular", wrong=0.3, seed=7)]
    for k in range(10):
        model = "equirectangular" if k % 3 == 2 else "perspective"
        ps_.append(pp.problem(20 + 97 * k, model=model, wrong=0.1 + 0.03 * k, noise=1e-3 * (k % 2), seed=10 + k))
    return ps_


@pytest.mark.parametrize("recompute,max_iter", [(True, 30), (False, 30), (True, 0)])
def test_batch_equals_single_calls_and_oracle(ps, recompute, max_iter):
    probs = _mixed()
    seeds = [17 * b + 3 for b in range(len(probs))]
    g = _solve(probs, 10, max_iter, recompute, seeds)
    for b, p in enumerate(probs):
        one = _solve([p], 10, max_iter, recompute, [seeds[b]])[0]
        _same(g[b], one)
        _same(g[b], _oracle(ps, p, 10, max_iter, recompute, seeds[b]))
        n = len(p["scale_factor"])
        if n < 10 or max_iter == 0:
            assert not g[b]["valid"] and g[b]["best_iter"] == -1 and np.array_equal(g[b]["pose_cw"], IDENTITY)


def test_noise_free_problems_return_the_true_pose():
    probs = [pp.problem(n, model=m, wrong=0.25, seed=50 + n) for n in (40, 200, 1500) for m in ("perspective", "equirectangular")]
    for g, p in zip(_solve(probs, 10, 30, True, list(range(len(probs)))), probs):
        assert g["valid"] and np.abs(g["pose_cw"] - p["pose_true"]).max() <= 1e-9
        assert np.array_equal(g["inliers"], ~p["bad"])


def test_repeated_calls_are_bit_identical():
    from openvslam_b200 import solve
    probs = [pp.problem(4000, model="equirectangular", noise=1e-3, seed=21), pp.problem(1000, noise=1e-3, seed=22)]
    s = solve.pnp_solver(10)
    a = s.find_via_ransac([pp.gpu_problem(p) for p in probs], 30, True, [1, 2])
    b = s.find_via_ransac([pp.gpu_problem(p) for p in probs], 30, True, [1, 2])
    s.close()
    for x, y in zip(a, b):
        _same(x, y)


def test_valid_exactly_when_the_best_count_reaches_min_num_inliers(ps):
    p = pp.problem(200, wrong=0.35, noise=1e-3, seed=40)
    c = _oracle(ps, p, 10, 30, False, 9)["num_inliers"]
    for m in (c - 1, c, c + 1):
        for recompute in (False, True):
            g = _solve([p], m, 30, recompute, [9])[0]
            _same(g, _oracle(ps, p, m, 30, recompute, 9))
            assert g["valid"] == (c >= m)
            if not recompute:
                assert g["num_inliers"] == c


def test_invalid_arguments_and_calls_without_a_launch():
    from openvslam_b200 import solve, _lib
    s = solve.pnp_solver(10)
    p = pp.gpu_problem(pp.problem(30, seed=1))
    before = _lib.launch_count()
    assert s.find_via_ransac([]) == []
    out = s.find_via_ransac([dict(bearings=np.zeros((0, 3)), pos_w=np.zeros((0, 3)), scale_factor=np.zeros(0, np.float32))])
    assert _lib.launch_count() == before
    assert not out[0]["valid"] and out[0]["best_iter"] == -1 and np.array_equal(out[0]["pose_cw"], IDENTITY)
    b2 = p["bearings"].copy(); b2[3] *= 1.001
    w2 = p["pos_w"].copy(); w2[4, 1] = np.inf
    b3 = p["bearings"].copy(); b3[0, 0] = np.nan
    for bad in (dict(bearings=b2), dict(pos_w=w2), dict(bearings=b3), dict(scale_factor=np.full(30, 0.0, np.float32)),
                dict(scale_factor=np.full(30, 90.5, np.float32)), dict(scale_factor=np.full(30, np.nan, np.float32))):
        with pytest.raises(_lib.OvsError) as e:
            s.find_via_ransac([dict(p, **bad)])
        assert e.value.code == -1
    with pytest.raises(_lib.OvsError):
        s.find_via_ransac([p], max_num_iter=-1)
    neg = solve.pnp_solver(-1)
    with pytest.raises(_lib.OvsError):
        neg.find_via_ransac([p])
    neg.close()
    s.close()


def test_invalidates_a_prepared_local_ba_on_the_same_handle():
    from openvslam_b200 import optimize, solve, synth, _lib
    q = synth.ba_problem(6, 2, 300, model="equirectangular", seed=6)
    prep = optimize.prepared_local_ba(optimize.camera(**q["cam"]), True, q["poses"], q["fixed"], q["points"], q["obs_kf"], q["obs_lm"],
                                      q["obs_xy"], None, q["inv_sigma_sq"])
    prep.run()
    p = pp.problem(100, seed=8)
    view = types.SimpleNamespace(_h=prep._h, min_num_inliers_=10)
    out = solve.pnp_solver.find_via_ransac(view, [pp.gpu_problem(p)], 30, True, [3])
    assert out[0]["valid"] and out[0]["num_inliers"] >= 70
    with pytest.raises(_lib.OvsError) as e:
        prep.run()
    assert e.value.code == -1   # OVS_ERR_INVALID_ARG
    prep.close()


def test_class_layer_adapter_recovers_the_true_pose(tmp_path):
    from openvslam_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_pnp_solver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "tests", "cpp", "standin"),
                           os.path.join(root, "tests", "cpp", "test_pnp_solver.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "pnp solver ok" in r.stdout, r.stdout + r.stderr
