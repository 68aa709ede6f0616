"""solve::sim3_solver on the GPU (k_sim3_ransac_prep + k_sim3_ransac: two launches per batch) against the oracle
(oracle/sim3_solver_oracle.c) and ground truth.  The kernel gives every hypothesis a warp whose lanes take the pairs with a stride
of 32, puts 4 hypotheses in a CTA and prepares the pairs in blocks of 256 threads; the sizes below sit around those strides."""
import os
import subprocess
import types

import numpy as np
import pytest

import sim3_ransac_problems as rp

pytestmark = pytest.mark.gpu

CONFIGS = [("perspective", False), ("perspective", True), ("equirectangular", False)]
SIZES = [3, 20, 31, 32, 33, 150, 255, 256, 257, 1000, 4000]
IDENTITY = np.concatenate([np.eye(3).ravel(), [0, 0, 0], [1.0]])


@pytest.fixture(scope="module")
def ss(oracle):
    """the solver's oracle (oracle/sim3_solver.py); `oracle` builds liboracle.so"""
    from oracle import sim3_solver
    return sim3_solver


def _oracle(ss, p, fix_scale, min_num_inliers, max_num_iter, seed):
    cam = ss.camera(**p["cam"])
    return ss.sim3_solve_ransac(cam, cam, *rp.args(p), fix_scale=fix_scale, min_num_inliers=min_num_inliers, max_num_iter=max_num_iter,
                                seed=seed)


def _same(g, o):
    assert g["valid"] == o["valid"]
    assert g["num_inliers"] == o["num_inliers"] and g["best_iter"] == o["best_iter"]
    assert np.array_equal(g["inliers"], o["inliers"])
    assert np.array_equal(g["sim3_12"], o["sim3_12"], equal_nan=True)


def _solve(problems, fix_scale, min_num_inliers=20, max_num_iter=200, seeds=None):
    from openvslam_b200 import solve
    s = solve.sim3_solver(fix_scale, min_num_inliers)
    out = s.find_via_ransac([rp.gpu_problem(p) for p in problems], max_num_iter, seeds)
    s.close()
    return out


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("model,fix_scale", CONFIGS)
def test_equals_oracle(ss, model, fix_scale, n):
    wrong = 0.1 + 0.3 * ((7 * n) % 10) / 10.0
    noise = 0.0 if n % 2 == 0 else 0.01
    p = rp.problem(n, model=model, fix_scale=fix_scale, wrong=wrong if n > 3 else 0.0, noise3d=noise, seed=n,
                   behind=n // 50 if model == "perspective" else 0)
    min_inl = max(1, min(20, n // 2))
    g = _solve([p], fix_scale, min_inl, 200, [1000 + n])[0]
    o = _oracle(ss, p, fix_scale, min_inl, 200, 1000 + n)
    _same(g, o)
    assert g["valid"] and g["num_inliers"] >= 0.5 * n
    if fix_scale:
        assert g["sim3_12"][12] == 1.0
    if noise == 0.0:
        assert np.abs(g["sim3_12"] - p["S_true"]).max() <= 1e-9


@pytest.mark.parametrize("max_num_iter", [1, 3, 4, 5, 7, 8, 9, 201])
def test_hypothesis_block_boundaries(ss, max_num_iter):
    p = rp.problem(100, wrong=0.4, noise3d=0.01, seed=31)
    g = _solve([p], False, 10, max_num_iter, [5])[0]
    _same(g, _oracle(ss, p, False, 10, max_num_iter, 5))


def _mixed(fix_scale):
    """16 problems: no pair, 2 pairs, fewer pairs than min_num_inliers (20), points behind camera 2, both camera models, noisy and
    exact, 10-40 % wrong"""
    ps = [rp.problem(0, seed=1), rp.problem(2, seed=2), rp.problem(10, seed=3, wrong=0.0), rp.problem(19, seed=4, wrong=0.1),
          rp.problem(300, seed=5, behind=40), rp.problem(60, model="equirectangular", fix_scale=fix_scale, seed=6, wrong=0.4)]
    for k in range(10):
        model = "equirectangular" if k % 3 == 2 else "perspective"
        ps.append(rp.problem(20 + 37 * k, model=model, fix_scale=fix_scale, wrong=0.1 + 0.03 * k, noise3d=0.01 * (k % 2), seed=10 + k,
                             behind=3 * (k % 2) if model == "perspective" else 0))
    return ps


def _degenerate(fix_scale):
    """min_num_inliers 3: coincident and collinear triples, and exact / wrong problems around them"""
    ps = [rp.degenerate("coincident", fix_scale=fix_scale, seed=1), rp.degenerate("collinear", fix_scale=fix_scale, seed=2),
          rp.degenerate("coincident", model="equirectangular", fix_scale=fix_scale, seed=3), rp.problem(3, seed=4, wrong=0.0),
          rp.problem(40, seed=5, behind=4)]
    return ps


@pytest.mark.parametrize("fix_scale", [False, True])
@pytest.mark.parametrize("batch,min_inl,max_iter", [("mixed", 20, 200), ("mixed", 20, 0), ("degenerate", 3, 50)])
def test_batch_equals_single_calls_and_oracle(ss, fix_scale, batch, min_inl, max_iter):
    ps = _mixed(fix_scale) if batch == "mixed" else _degenerate(fix_scale)
    seeds = [17 * b + 3 for b in range(len(ps))]
    g = _solve(ps, fix_scale, min_inl, max_iter, seeds)
    for b, p in enumerate(ps):
        one = _solve([p], fix_scale, min_inl, max_iter, [seeds[b]])[0]
        _same(g[b], one)
        _same(g[b], _oracle(ss, p, fix_scale, min_inl, max_iter, seeds[b]))
        n = len(p["sigma_sq_1"])
        if n < 3 or n < min_inl or max_iter == 0:
            assert not g[b]["valid"] and g[b]["best_iter"] == -1 and np.array_equal(g[b]["sim3_12"], IDENTITY)
    if batch == "degenerate" and not fix_scale:
        assert g[0]["best_iter"] == -1 and g[0]["num_inliers"] == 0   # a coincident triple's 0 / 0 scale scores nothing


def test_repeated_calls_are_bit_identical():
    from openvslam_b200 import solve
    ps = [rp.problem(4000, model="equirectangular", seed=21), rp.problem(1000, seed=22, noise3d=0.01)]
    s = solve.sim3_solver(False)
    a = s.find_via_ransac([rp.gpu_problem(p) for p in ps], 200, [1, 2])
    b = s.find_via_ransac([rp.gpu_problem(p) for p in ps], 200, [1, 2])
    s.close()
    for x, y in zip(a, b):
        _same(x, y)


def test_valid_exactly_when_the_best_count_reaches_min_num_inliers(ss):
    p = rp.problem(200, wrong=0.35, noise3d=0.01, seed=40)
    o = _oracle(ss, p, False, 20, 200, 9)
    c = o["num_inliers"]
    for m in (c - 1, c, c + 1):
        g = _solve([p], False, m, 200, [9])[0]
        om = _oracle(ss, p, False, m, 200, 9)
        _same(g, om)
        assert g["valid"] == (c >= m) and g["num_inliers"] == c


def test_invalid_arguments_and_calls_without_a_launch():
    from openvslam_b200 import solve, _lib
    s = solve.sim3_solver(False)
    p = rp.gpu_problem(rp.problem(30, seed=1))
    before = _lib.launch_count()
    assert s.find_via_ransac([]) == []
    out = s.find_via_ransac([dict(p, pos_w_1=np.zeros((0, 3)), pos_w_2=np.zeros((0, 3)), sigma_sq_1=np.zeros(0), sigma_sq_2=np.zeros(0))])
    assert _lib.launch_count() == before
    assert not out[0]["valid"] and out[0]["best_iter"] == -1 and np.array_equal(out[0]["sim3_12"], IDENTITY)
    for bad in (dict(sigma_sq_1=np.full(30, -1.0, np.float32)), dict(sigma_sq_2=np.full(30, np.nan, np.float32)),
                dict(sigma_sq_1=np.full(30, np.inf, np.float32))):
        with pytest.raises(_lib.OvsError) as e:
            s.find_via_ransac([dict(p, **bad)])
        assert e.value.code == -1
    from openvslam_b200 import optimize
    cam = optimize.camera(**rp.problem(3, seed=1)["cam"])
    cam.model = 7
    with pytest.raises(_lib.OvsError):
        s.find_via_ransac([dict(p, cam_2=cam)])
    with pytest.raises(_lib.OvsError):
        s.find_via_ransac([p], max_num_iter=-1)
    neg = solve.sim3_solver(False, -1)
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
    p = rp.problem(100, seed=8)
    view = types.SimpleNamespace(_h=prep._h, fix_scale_=False, min_num_inliers_=20)
    out = solve.sim3_solver.find_via_ransac(view, [rp.gpu_problem(p)], 200, [3])
    assert out[0]["valid"] and out[0]["num_inliers"] >= 70
    with pytest.raises(_lib.OvsError) as e:
        prep.run()
    assert e.value.code == -1   # OVS_ERR_INVALID_ARG
    prep.close()


def test_class_layer_adapter_recovers_the_true_sim3(tmp_path):
    from openvslam_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_sim3_solver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "tests", "cpp", "standin"),
                           os.path.join(root, "tests", "cpp", "test_sim3_solver.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "sim3 solver ok" in r.stdout, r.stdout + r.stderr
