"""solve::homography_solver and solve::fundamental_solver on the GPU (k_two_view_normalize + k_two_view_hypotheses +
k_two_view_score + k_two_view_refine: four launches per batch) against the oracle (oracle/two_view_solver_oracle.c) and ground
truth.  The kernels give every hypothesis one thread for the minimal solve and then a warp whose lanes take the matches with a
stride of 32, put 4 hypotheses in a CTA, and recompute with one 256-thread CTA per problem whose sums take 256 strided partials;
the sizes below sit around those strides."""
import os
import subprocess
import types

import numpy as np
import pytest

import two_view_problems as tp

pytestmark = pytest.mark.gpu

SIZES = [8, 9, 31, 32, 33, 255, 256, 257, 1000, 4000]
MODELS = ["H", "F"]
KEY = {"H": "H_21", "F": "F_21"}


@pytest.fixture(scope="module")
def tv(oracle):
    """the solvers' oracle (oracle/two_view_solver.py); `oracle` builds liboracle.so"""
    from oracle import two_view_solver
    return two_view_solver


def _oracle(tv, model, p, max_num_iter, recompute, seed):
    return tv.solve_ransac(model, p["keypts_1"], p["keypts_2"], p["matches_12"], max_num_iter, recompute=recompute, seed=seed)


def _same(g, o, model):
    assert g["valid"] == o["valid"]
    assert g["num_inliers"] == o["num_inliers"] and g["best_iter"] == o["best_iter"]
    assert np.array_equal(g["inliers"], o["inliers"])
    M = o["M"] if "M" in o else o[KEY[model]]
    assert np.array_equal(g[KEY[model]], M, equal_nan=True)
    assert np.array_equal(np.float64(g["best_score"]), np.float64(o["best_score"]), equal_nan=True)


def _solver(model, h=None):
    from openvslam_b200 import solve
    cls = solve.homography_solver if model == "H" else solve.fundamental_solver
    return cls()


def _solve(model, problems, max_num_iter=100, recompute=True, seeds=None):
    s = _solver(model)
    out = s.find_via_ransac([tp.gpu_problem(p) for p in problems], max_num_iter, recompute, seeds)
    s.close()
    return out


@pytest.mark.parametrize("recompute", [True, False])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("model", MODELS)
def test_equals_oracle(tv, model, n, recompute):
    wrong = 0.4 * ((7 * n) % 11) / 10.0
    noise = 0.0 if n % 2 == 0 else 1.0
    scene = "planar" if (model == "H") == (n % 3 != 0) else "general"
    p = tp.problem(n, scene=scene, wrong=wrong, noise=noise, seed=n)
    g = _solve(model, [p], 100, recompute, [1000 + n])[0]
    _same(g, _oracle(tv, model, p, 100, recompute, 1000 + n), model)


@pytest.mark.parametrize("max_num_iter", [0, 1, 3, 4, 5, 100, 201])
@pytest.mark.parametrize("model", MODELS)
def test_hypothesis_block_boundaries(tv, model, max_num_iter):
    p = tp.problem(300, scene="planar", wrong=0.3, noise=1.0, seed=31)
    for recompute in (True, False):
        g = _solve(model, [p], max_num_iter, recompute, [5])[0]
        _same(g, _oracle(tv, model, p, max_num_iter, recompute, 5), model)
        if max_num_iter == 0:
            assert not g["valid"] and g["best_iter"] == -1 and not g[KEY[model]].any()


@pytest.mark.parametrize("model", MODELS)
def test_noise_free_problems_make_every_correct_match_an_inlier(model):
    scene = "planar" if model == "H" else "general"
    probs = [tp.problem(n, scene=scene, wrong=0.0, seed=50 + n) for n in (40, 200, 1500)]
    for g, p in zip(_solve(model, probs, 100, True, list(range(len(probs)))), probs):
        assert g["valid"] and g["inliers"].all()
        c1, c2 = tp.chis(model, g[KEY[model]], p["keypts_1"], p["keypts_2"], p["matches_12"])
        assert np.sqrt(np.maximum(c1, c2)).max() < 1e-3   # transfer / epipolar distance in px (sigma = 1)


def _mixed():
    """0, 7 and exactly 8 matches, coincident and collinear keypoints, a planar scene (degenerate for F), pure rotation, n1 != n2,
    noisy and exact, 0-40 % wrong"""
    ps_ = [tp.problem(0, seed=1), tp.problem(7, wrong=0.0, seed=2), tp.problem(8, wrong=0.0, seed=3),
           tp.degenerate("coincident", seed=4), tp.degenerate("collinear", seed=5), tp.degenerate("planar", seed=6),
           tp.degenerate("rotation", seed=7), tp.problem(300, scene="planar", wrong=0.3, seed=8, n1=900, n2=350)]
    for k in range(10):
        scene = "planar" if k % 3 == 2 else "general"
        ps_.append(tp.problem(20 + 97 * k, scene=scene, wrong=0.04 * k, noise=1.0 * (k % 2), seed=10 + k, n2=40 + 130 * k))
    return ps_


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("recompute,max_iter", [(True, 100), (False, 100), (True, 0)])
def test_batch_equals_single_calls_and_oracle(tv, model, recompute, max_iter):
    probs = _mixed()
    seeds = [17 * b + 3 for b in range(len(probs))]
    g = _solve(model, probs, max_iter, recompute, seeds)
    for b, p in enumerate(probs):
        one = _solve(model, [p], max_iter, recompute, [seeds[b]])[0]
        _same(g[b], one, model)
        _same(g[b], _oracle(tv, model, p, max_iter, recompute, seeds[b]), model)
        if len(p["matches_12"]) < 8 or max_iter == 0:
            assert not g[b]["valid"] and g[b]["best_iter"] == -1 and not g[b][KEY[model]].any()


@pytest.mark.parametrize("model", MODELS)
def test_repeated_calls_are_bit_identical(model):
    probs = [tp.problem(4000, scene="planar", wrong=0.2, noise=1.0, seed=21), tp.problem(1000, wrong=0.1, noise=1.0, seed=22)]
    s = _solver(model)
    a = s.find_via_ransac([tp.gpu_problem(p) for p in probs], 100, True, [1, 2])
    b = s.find_via_ransac([tp.gpu_problem(p) for p in probs], 100, True, [1, 2])
    s.close()
    for x, y in zip(a, b):
        _same(x, dict(y, M=y[KEY[model]]), model)


# (offset in px of the last match's view-2 keypoint, seed) of 8-match problems whose best hypothesis has 7 and 8 inliers
FLIP_CASES = {"H": {7: (4.0, 1), 8: (4.0, 0)}, "F": {7: (6.0, 4), 8: (4.0, 4)}}


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("count", [7, 8])
def test_valid_flips_exactly_at_8_inliers(tv, model, count):
    """8 matches, 7 of them exact, the last one's view-2 keypoint moved: the best hypothesis has `count` inliers and a positive
    score (asserted on the oracle), and valid is set exactly when count >= 8"""
    d, seed = FLIP_CASES[model][count]
    p = tp.problem(8, scene="planar" if model == "H" else "general", wrong=0.0, seed=seed, n1=60, n2=60)
    k2 = p["keypts_2"].copy()
    k2[p["matches_12"][7, 1], 1] += np.float32(d)
    q = dict(p, keypts_2=k2)
    o = _oracle(tv, model, q, 100, False, 9)
    assert o["best_iter"] >= 0 and o["best_score"] > 0 and o["num_inliers"] == count
    g = _solve(model, [q], 100, False, [9])[0]
    _same(g, o, model)
    assert g["valid"] == (count >= 8)


@pytest.mark.parametrize("model", MODELS)
def test_invalid_arguments_and_calls_without_a_launch(model):
    from openvslam_b200 import solve, _lib
    s = _solver(model)
    p = tp.gpu_problem(tp.problem(30, seed=1))
    before = _lib.launch_count()
    assert s.find_via_ransac([], 100) == []
    out = s.find_via_ransac([dict(keypts_1=p["keypts_1"], keypts_2=p["keypts_2"], matches_12=np.zeros((0, 2), np.int32))], 100)
    assert _lib.launch_count() == before
    assert not out[0]["valid"] and out[0]["best_iter"] == -1 and not out[0][KEY[model]].any()
    k1 = p["keypts_1"].copy(); k1[4, 0] = np.nan
    k2 = p["keypts_2"].copy(); k2[2, 1] = np.inf
    m_hi = p["matches_12"].copy(); m_hi[3, 1] = len(p["keypts_2"])
    m_neg = p["matches_12"].copy(); m_neg[0, 0] = -1
    for bad in (dict(keypts_1=k1), dict(keypts_2=k2), dict(matches_12=m_hi), dict(matches_12=m_neg)):
        with pytest.raises(_lib.OvsError) as e:
            s.find_via_ransac([dict(p, **bad)], 100)
        assert e.value.code == -1
    with pytest.raises(_lib.OvsError):
        s.find_via_ransac([p], -1)
    s.close()
    for sigma in (0.0, -1.0):
        bad_s = (solve.homography_solver if model == "H" else solve.fundamental_solver)(sigma=sigma)
        with pytest.raises(_lib.OvsError) as e:
            bad_s.find_via_ransac([p], 100)
        assert e.value.code == -1
        bad_s.close()
    assert _lib.launch_count() == before


def test_a_call_is_four_launches():
    from openvslam_b200 import _lib
    p = tp.problem(200, scene="planar", wrong=0.2, seed=3)
    for model in MODELS:
        s = _solver(model)
        s.find_via_ransac([tp.gpu_problem(p)] * 3, 100)
        before = _lib.launch_count()
        s.find_via_ransac([tp.gpu_problem(p)] * 3, 100)
        assert _lib.launch_count() - before == 4
        before = _lib.launch_count()
        s.find_via_ransac([tp.gpu_problem(p)] * 3, 0)
        assert _lib.launch_count() - before == 1
        s.close()


def test_brute_force_and_essential_on_the_same_handle_are_unaffected_by_solves():
    import essential_problems as ep
    from openvslam_b200 import match, solve
    rng = np.random.default_rng(12)
    d1 = rng.integers(0, 256, (400, 32), dtype=np.uint8)
    d2 = d1[rng.permutation(400)[:350]].copy()
    r = match.robust(0.8, False)
    a = r.brute_force_match(d1, d2, None)
    e = ep.problem(1000, wrong=0.2, noise=1e-3, seed=13)
    view = types.SimpleNamespace(_h=r._h)
    ea = solve.essential_solver.find_via_ransac(view, [ep.gpu_problem(e)], 50, True, [4])
    p = tp.problem(4000, scene="planar", wrong=0.2, noise=1.0, seed=13)
    for cls in (solve.homography_solver, solve.fundamental_solver):
        out = cls.find_via_ransac(types.SimpleNamespace(_h=r._h, sigma_=1.0, _entry=cls._entry, _key=cls._key), [tp.gpu_problem(p)], 201, True, [4])
        assert out[0]["valid"]
    b = r.brute_force_match(d1, d2, None)
    eb = solve.essential_solver.find_via_ransac(view, [ep.gpu_problem(e)], 50, True, [4])
    assert np.array_equal(a, b)
    assert np.array_equal(ea[0]["E_21"], eb[0]["E_21"]) and np.array_equal(ea[0]["inliers"], eb[0]["inliers"])
    r.close()


def test_class_layer_adapters_recover_the_truth(tmp_path):
    from openvslam_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_two_view_solvers")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "tests", "cpp", "standin"),
                           os.path.join(root, "tests", "cpp", "test_two_view_solvers.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "two-view solvers ok" in r.stdout, r.stdout + r.stderr
