"""solve::essential_solver and match::robust::match_frame_and_keyframe on the GPU (k_two_view_hypotheses + k_two_view_score +
k_two_view_refine instantiated for EssentialModel: three launches per batch) against the oracle (oracle/essential_solver_oracle.c) and ground truth.  The kernels
give every hypothesis one thread for the eight-point E and then a warp whose lanes take the matches with a stride of 32, put 4
hypotheses in a CTA, and recompute with one 256-thread CTA per problem whose sums take 256 strided partials; the sizes below sit
around those strides."""
import os
import subprocess
import types

import numpy as np
import pytest

import essential_problems as ep

pytestmark = pytest.mark.gpu

SIZES = [8, 9, 31, 32, 33, 255, 256, 257, 1000, 4000]


@pytest.fixture(scope="module")
def es(oracle):
    """the solver's oracle (oracle/essential_solver.py); `oracle` builds liboracle.so"""
    from oracle import essential_solver
    return essential_solver


def _oracle(es, p, max_num_iter, recompute, seed):
    return es.essential_solve_ransac(p["bearings_1"], p["bearings_2"], max_num_iter, recompute=recompute, seed=seed)


def _same(g, o):
    assert g["valid"] == o["valid"]
    assert g["num_inliers"] == o["num_inliers"] and g["best_iter"] == o["best_iter"]
    assert np.array_equal(g["inliers"], o["inliers"])
    assert np.array_equal(g["E_21"], o["E_21"], equal_nan=True)
    assert np.array_equal(np.float64(g["best_score"]), np.float64(o["best_score"]), equal_nan=True)


def _solve(problems, max_num_iter=50, recompute=True, seeds=None):
    from openvslam_b200 import solve
    s = solve.essential_solver()
    out = s.find_via_ransac([ep.gpu_problem(p) for p in problems], max_num_iter, recompute, seeds)
    s.close()
    return out


def _unit_E(E):
    return E / np.linalg.norm(E)


def _close_up_to_sign(a, b, tol):
    return min(np.abs(a - b).max(), np.abs(a + b).max()) <= tol


@pytest.mark.parametrize("recompute", [True, False])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("model", ["perspective", "equirectangular"])
def test_equals_oracle(es, model, n, recompute):
    wrong = 0.4 * ((7 * n) % 11) / 10.0
    noise = 0.0 if n % 2 == 0 else 1e-3
    p = ep.problem(n, model=model, wrong=wrong, noise=noise, seed=n)
    g = _solve([p], 50, recompute, [1000 + n])[0]
    _same(g, _oracle(es, p, 50, recompute, 1000 + n))


@pytest.mark.parametrize("max_num_iter", [0, 1, 3, 4, 5, 50, 51, 201])
def test_hypothesis_block_boundaries(es, max_num_iter):
    p = ep.problem(300, model="equirectangular", wrong=0.3, noise=1e-3, seed=31)
    for recompute in (True, False):
        g = _solve([p], max_num_iter, recompute, [5])[0]
        _same(g, _oracle(es, p, max_num_iter, recompute, 5))
        if max_num_iter == 0:
            assert not g["valid"] and g["best_iter"] == -1 and not g["E_21"].any()


def test_noise_free_problems_return_the_true_E():
    probs = [ep.problem(n, model=m, wrong=0.0, seed=50 + n) for n in (40, 200, 1500) for m in ("perspective", "equirectangular")]
    for g, p in zip(_solve(probs, 50, True, list(range(len(probs)))), probs):
        assert g["valid"] and g["inliers"].all()
        assert _close_up_to_sign(_unit_E(g["E_21"]), _unit_E(p["E_true"]), 1e-9)


def _mixed():
    """0, 7 and exactly 8 matches, coincident and collinear bearings, pure rotation, a planar scene, both bearing types, noisy and
    exact, 0-40 % wrong"""
    ps_ = [ep.problem(0, seed=1), ep.problem(7, wrong=0.0, seed=2), ep.problem(8, wrong=0.0, seed=3),
           ep.degenerate("coincident", seed=4), ep.degenerate("collinear", seed=5), ep.degenerate("planar", seed=6),
           ep.degenerate("rotation", seed=7), ep.problem(300, model="equirectangular", wrong=0.3, seed=8)]
    for k in range(10):
        model = "equirectangular" if k % 3 == 2 else "perspective"
        ps_.append(ep.problem(20 + 97 * k, model=model, wrong=0.04 * k, noise=1e-3 * (k % 2), seed=10 + k))
    return ps_


@pytest.mark.parametrize("recompute,max_iter", [(True, 50), (False, 50), (True, 0)])
def test_batch_equals_single_calls_and_oracle(es, recompute, max_iter):
    probs = _mixed()
    seeds = [17 * b + 3 for b in range(len(probs))]
    g = _solve(probs, max_iter, recompute, seeds)
    for b, p in enumerate(probs):
        one = _solve([p], max_iter, recompute, [seeds[b]])[0]
        _same(g[b], one)
        _same(g[b], _oracle(es, p, max_iter, recompute, seeds[b]))
        n = len(p["bearings_1"])
        if n < 8 or max_iter == 0:
            assert not g[b]["valid"] and g[b]["best_iter"] == -1 and not g[b]["E_21"].any()


@pytest.mark.parametrize("view", ["strided", "reversed"])
def test_seeds_given_as_a_view_equal_their_contiguous_copy(view):
    """seeds may be any 1-D array: a strided or reversed view gives the result of its values, not of the memory it starts at"""
    probs = [ep.problem(300, model=m, wrong=0.4, noise=1e-3, seed=60 + k) for k, m in enumerate(["perspective", "equirectangular"] * 2)]
    base = np.arange(100, 100 + 2 * len(probs), dtype=np.uint64)
    seeds = base[::2] if view == "strided" else base[len(probs):][::-1]
    g = _solve(probs, 50, True, seeds)
    for x, y in zip(g, _solve(probs, 50, True, np.array(seeds))):
        _same(x, y)
    if view == "strided":   # the seeds make a difference here: reading the view's memory as if contiguous would be seen
        assert any(x["best_iter"] != y["best_iter"] or not np.array_equal(x["inliers"], y["inliers"])
                   for x, y in zip(g, _solve(probs, 50, True, base[:len(probs)])))


def test_repeated_calls_are_bit_identical():
    from openvslam_b200 import solve
    probs = [ep.problem(4000, model="equirectangular", wrong=0.2, noise=1e-3, seed=21), ep.problem(1000, wrong=0.1, noise=1e-3, seed=22)]
    s = solve.essential_solver()
    a = s.find_via_ransac([ep.gpu_problem(p) for p in probs], 50, True, [1, 2])
    b = s.find_via_ransac([ep.gpu_problem(p) for p in probs], 50, True, [1, 2])
    s.close()
    for x, y in zip(a, b):
        _same(x, y)


def test_invalid_arguments_and_calls_without_a_launch():
    from openvslam_b200 import solve, _lib
    s = solve.essential_solver()
    p = ep.gpu_problem(ep.problem(30, seed=1))
    before = _lib.launch_count()
    assert s.find_via_ransac([], 50) == []
    out = s.find_via_ransac([dict(bearings_1=np.zeros((0, 3)), bearings_2=np.zeros((0, 3)))], 50)
    assert _lib.launch_count() == before
    assert not out[0]["valid"] and out[0]["best_iter"] == -1 and not out[0]["E_21"].any()
    b2 = p["bearings_2"].copy(); b2[3] *= 1.001
    b1 = p["bearings_1"].copy(); b1[0, 0] = np.nan
    b3 = p["bearings_1"].copy(); b3[7, 2] = np.inf
    for bad in (dict(bearings_2=b2), dict(bearings_1=b1), dict(bearings_1=b3)):
        with pytest.raises(_lib.OvsError) as e:
            s.find_via_ransac([dict(p, **bad)], 50)
        assert e.value.code == -1
    with pytest.raises(_lib.OvsError):
        s.find_via_ransac([p], -1)
    s.close()


# ------------------------------------------------------------------ match::robust::match_frame_and_keyframe
def _views(n1, n2, m, model="perspective", seed=0, wrong=0.2):
    """a frame (camera 1) with n1 keypoints and a keyframe (camera 2) with n2: m frame keypoints carry a keyframe descriptor with
    0..6 bits flipped; `wrong` of those get the bearing of another point (so that their pair breaks the geometry); the rest are
    random.  lm_valid_2: 90 % of the keyframe keypoints."""
    rng = np.random.default_rng(seed)
    p = ep.problem(max(n1, n2), model=model, wrong=0.0, seed=seed)
    desc_kf = rng.integers(0, 256, (n2, 32), dtype=np.uint8)
    desc_frm = rng.integers(0, 256, (n1, 32), dtype=np.uint8)
    src = rng.choice(n2, m, replace=False)             # keyframe keypoint of frame keypoint dst[k]
    dst = rng.choice(n1, m, replace=False)
    b_kf = p["bearings_2"][:n2].copy()
    b_frm = ep._unit(rng.normal(size=(n1, 3)))
    for k in range(m):
        desc_frm[dst[k]] = desc_kf[src[k]]
        for _ in range(rng.integers(0, 7)):
            bit = rng.integers(0, 256)
            desc_frm[dst[k], bit // 8] ^= np.uint8(1 << (bit % 8))
        b_frm[dst[k]] = p["bearings_1"][src[k]]
    nw = int(wrong * m)
    for k in range(nw):
        b_frm[dst[k]] = p["bearings_1"][src[(k + 1) % m]]
    lm_valid = (rng.random(n2) < 0.9).astype(np.uint8)
    return dict(desc_frm=desc_frm, b_frm=np.ascontiguousarray(b_frm), desc_kf=desc_kf, b_kf=np.ascontiguousarray(b_kf), lm_valid=lm_valid)


def _match_host(v, seed=0, max_num_iter=50, m=None):
    from openvslam_b200 import match
    r = m or match.robust(0.8, False)
    out = r.match_frame_and_keyframe(v["desc_frm"], v["b_frm"], v["desc_kf"], v["b_kf"], v["lm_valid"], max_num_iter, seed)
    if m is None:
        r.close()
    return out


@pytest.mark.parametrize("model,n1,n2,m", [("perspective", 300, 280, 200), ("equirectangular", 1500, 1200, 900), ("perspective", 40, 30, 12)])
def test_composed_matcher_equals_oracle_and_device_twin(es, model, n1, n2, m):
    import torch
    from openvslam_b200 import match
    from oracle import oracle as O
    v = _views(n1, n2, m, model=model, seed=n1)
    r = match.robust(0.8, False)
    num, idx = _match_host(v, seed=9, m=r)
    onum, oidx = es.robust_match_frame_and_keyframe(v["desc_frm"], v["b_frm"], v["desc_kf"], v["b_kf"], v["lm_valid"], 0.8, 50, 9)
    assert num == onum and np.array_equal(idx, oidx)
    # the pairs are the brute force's, bit for bit, and every inlier is one of them
    pairs = r.brute_force_match(v["desc_frm"], v["desc_kf"], v["lm_valid"])
    assert np.array_equal(pairs, O.robust_brute_force_match(v["desc_frm"], v["desc_kf"], v["lm_valid"], 0.8))
    sel = idx >= 0
    assert set(zip(np.flatnonzero(sel), idx[sel])) <= set(map(tuple, pairs))
    assert num == sel.sum() and (num == 0 or num >= 8)
    # the device twin on resident descriptors and bearings
    dev = [torch.from_numpy(a).cuda() for a in (v["desc_frm"], v["b_frm"], v["desc_kf"], v["b_kf"])]
    torch.cuda.synchronize()
    dnum, didx = r.match_frame_and_keyframe_device(dev[0].data_ptr(), dev[1].data_ptr(), n1, dev[2].data_ptr(), dev[3].data_ptr(), n2,
                                                   v["lm_valid"], 50, 9)
    assert dnum == num and np.array_equal(didx, idx)
    r.close()


def test_composed_matcher_with_fewer_than_8_pairs_matches_nothing():
    from openvslam_b200 import match, _lib
    v = _views(50, 40, 6, seed=3, wrong=0.0)
    r = match.robust(0.8, False)
    assert len(r.brute_force_match(v["desc_frm"], v["desc_kf"], v["lm_valid"])) < 8
    before = _lib.launch_count()
    num, idx = _match_host(v, m=r)
    launches = _lib.launch_count() - before
    assert num == 0 and (idx == -1).all()
    # only the brute force ran (its Hamming kernel and any re-queries): no solver launch
    r2 = match.robust(0.8, False)
    before = _lib.launch_count()
    r2.brute_force_match(v["desc_frm"], v["desc_kf"], v["lm_valid"])
    assert launches == _lib.launch_count() - before
    r.close(); r2.close()


def test_brute_force_on_the_same_handle_is_unchanged_by_a_solve():
    from openvslam_b200 import match, solve
    v = _views(400, 350, 300, seed=12)
    r = match.robust(0.8, False)
    a = r.brute_force_match(v["desc_frm"], v["desc_kf"], v["lm_valid"])
    view = types.SimpleNamespace(_h=r._h)
    p = ep.problem(4000, wrong=0.2, noise=1e-3, seed=13)
    out = solve.essential_solver.find_via_ransac(view, [ep.gpu_problem(p)], 201, True, [4])
    assert out[0]["valid"]
    b = r.brute_force_match(v["desc_frm"], v["desc_kf"], v["lm_valid"])
    assert np.array_equal(a, b)
    r.close()


def test_class_layer_adapters_recover_the_true_E_and_landmarks(tmp_path):
    from openvslam_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "test_essential_solver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "tests", "cpp", "standin"),
                           os.path.join(root, "tests", "cpp", "test_essential_solver.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "essential solver ok" in r.stdout, r.stdout + r.stderr
