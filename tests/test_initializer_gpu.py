"""GPU tests of monocular map initialisation (ovs_initialize_perspective_host, ovs_initialize_bearing_vector_host): every output
against the oracle (oracle/initializer_oracle.c) bit for bit, the statuses, the truth on noise-free scenes, batches against single
calls, the solvers inside the call against the standalone solver entry points, launch counts and argument checks."""
import ctypes as C

import numpy as np
import pytest

import initializer_problems as IP

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib_init():
    from openvslam_b200 import initialize, optimize
    return initialize, optimize


def _view(initialize, optimize, p, side):
    c = p["cam"]
    cam = optimize.Camera(c["model"], c["fx"], c["fy"], c["cx"], c["cy"], 0.0, c["cols"], c["rows"])
    return initialize.view(cam, p["keypts_" + side], p["bearings_" + side])


def _gpu(lib_init, problems, perspective, seeds=None, **kw):
    initialize, optimize = lib_init
    cls = initialize.perspective if perspective else initialize.bearing_vector
    h = cls(None, **kw)
    try:
        return h.initialize_batch([dict(ref=_view(initialize, optimize, p, "ref"), cur=_view(initialize, optimize, p, "cur"),
                                        ref_matches_with_cur=p["ref_matches_with_cur"]) for p in problems], seeds)
    finally:
        h.close()


def _oracle(p, seed, **kw):
    import oracle.initializer as OI
    args = dict(num_ransac_iters=kw.get("num_ransac_iters", 100), min_num_triangulated=kw.get("min_num_triangulated", 50),
                parallax_deg_thr=kw.get("parallax_deg_thr", 1.0), reproj_err_thr_sq=kw.get("reproj_err_thr_sq", 4.0), seed=seed)
    return OI.initialize(*IP.oracle_args(p), **args)


def _near_threshold(p, o, i_ref):
    """a reference keypoint whose decision under the chosen hypothesis sits within rounding of a check_pose threshold"""
    r = o["result"]
    c = p["ref_matches_with_cur"][i_ref]
    R = np.array(r.rot_ref_to_cur[:]).reshape(3, 3); t = np.array(r.trans_ref_to_cur[:])
    _, _, _, _, margin = IP.check_pose(R, t, p["cam"], p["cam"], p["bearings_ref"][[i_ref]], p["bearings_cur"][[c]],
                                       p["keypts_ref"][[i_ref]].astype(np.float64), p["keypts_cur"][[c]].astype(np.float64),
                                       np.ones(1, bool), depth_is_positive=p["perspective"])
    return margin[0] < 1e-9


def _assert_equal(p, g, o):
    r = o["result"]
    assert (g["status_code"], g["model"], g["chosen"], g["num_hypotheses"]) == (r.status, {0: None, 1: "H", 2: "F", 3: "E"}[r.model],
                                                                               r.chosen, r.num_hypotheses)
    assert np.array_equal(g["num_valid"], np.array(r.num_valid[:], np.int32))
    assert np.array_equal(g["cos_parallax"].view(np.uint32), np.array(r.cos_parallax[:], np.float32).view(np.uint32))
    assert np.array_equal(g["rot_ref_to_cur"].ravel(), np.array(r.rot_ref_to_cur[:]))
    assert np.array_equal(g["trans_ref_to_cur"], np.array(r.trans_ref_to_cur[:]))
    assert np.array_equal(g["solver_M"].reshape(2, 9), np.array([r.solver_M[s][:] for s in range(2)]))
    assert np.array_equal(g["solver_score"], np.array(r.solver_score[:]))
    assert np.array_equal(g["solver_num_inliers"], np.array(r.solver_num_inliers[:]))
    assert np.array_equal(g["solver_valid"], np.array(r.solver_valid[:], bool))
    diff = np.nonzero((g["is_triangulated"] != o["is_triangulated"]) | (g["triangulated_pts"] != o["triangulated_pts"]).any(1))[0]
    if p["perspective"]:
        assert len(diff) == 0, diff
    else:   # the equirectangular reprojection's atan2 / asin may round differently on the device
        assert all(_near_threshold(p, o, i) for i in diff), diff


CASES = [("planar", "perspective"), ("general", "perspective"), ("general", "equirect")]


@pytest.mark.parametrize("scene,camera", CASES)
@pytest.mark.parametrize("m", [8, 9, 255, 256, 257, 1000, 4000])
def test_equals_oracle(lib_init, scene, camera, m):
    problems = [IP.problem(m, scene=scene, camera=camera, wrong=w, noise=nz, seed=m + k)
                for k, (w, nz) in enumerate([(0.0, 0.0), (0.2, 1.0), (0.4, 1.0)])]
    seeds = [11, 12, 13]
    got = _gpu(lib_init, problems, camera == "perspective", seeds)
    for p, g, s in zip(problems, got, seeds):
        _assert_equal(p, g, _oracle(p, s))


@pytest.mark.parametrize("m", [49, 50, 51, 52])
def test_min_num_triangulated_and_rank_edges(lib_init, m):
    problems = [IP.problem(m, seed=s, extra=3) for s in range(3)] + [IP.problem(m, camera="equirect", seed=s, extra=3) for s in range(2)]
    statuses = set()
    for persp, sub in ((True, problems[:3]), (False, problems[3:])):
        got = _gpu(lib_init, sub, persp, [5] * len(sub))
        for p, g in zip(sub, got):
            _assert_equal(p, g, _oracle(p, 5))
            # noise-free and no wrong match: the best hypothesis keeps every match, so min_num_triangulated = 50 decides between
            # too few and the parallax test, and the parallax is the rank-min(50, n - 1) cosine of exactly m values
            assert g["num_valid"].max() == m, (g["num_valid"], m)
            assert g["status"] == "too few" if m < 50 else g["status"] in ("ok", "small parallax"), g["status"]
            statuses.add(g["status"])
    assert "ok" in statuses or m < 50


def _status_problems():
    return {"no valid model": IP.problem(7, seed=1), "decomposition refused": IP.problem(300, scene="rotation", seed=1),
            "too few": IP.problem(30, seed=1), "ambiguous": IP.problem(200, scene="planar", baseline=0.05, seed=0),
            "small parallax": IP.problem(300, baseline=0.002, seed=1), "ok": IP.problem(300, seed=1)}


def test_every_status(lib_init):
    ps = _status_problems()
    got = _gpu(lib_init, list(ps.values()), True, [0] * len(ps))
    for (name, p), g in zip(ps.items(), got):
        assert g["status"] == name
        _assert_equal(p, g, _oracle(p, 0))


@pytest.mark.parametrize("scene,camera", CASES)
def test_noise_free_truth(lib_init, scene, camera):
    """float32 keypoints bound the recovery: about 1e-7 for R and 1e-6 for t / |t|"""
    problems = [IP.problem(500, scene=scene, camera=camera, seed=s) for s in (1, 3, 4)]
    for p, g in zip(problems, _gpu(lib_init, problems, camera == "perspective")):
        assert g["ok"]
        assert np.abs(g["rot_ref_to_cur"] - p["R"]).max() <= 1e-6
        assert np.abs(g["trans_ref_to_cur"] - p["t"] / np.linalg.norm(p["t"])).max() <= 1e-5
        tri = g["is_triangulated"]
        truth = np.zeros((len(tri), 3)); truth[p["matched_ref"]] = p["p_ref"] / np.linalg.norm(p["t"])
        err = np.linalg.norm(g["triangulated_pts"][tri] - truth[tri], axis=1) / np.linalg.norm(truth[tri], axis=1)
        assert tri[p["matched_ref"]].mean() > 0.9 and err.max() <= 1e-3 and np.median(err) <= 1e-5


def test_batch_equals_single_calls_and_repeats(lib_init):
    ps = list(_status_problems().values())
    ps += [IP.problem(m, scene=sc, wrong=w, noise=1.0, seed=20 + k) for k, (m, sc, w) in
           enumerate([(300, "planar", 0.1), (700, "general", 0.3), (120, "planar", 0.0), (1500, "general", 0.2), (60, "general", 0.0)])]
    ps += [IP.problem(m, seed=40 + m, extra=m // 3) for m in (90, 400)]
    empty = IP.problem(20, seed=3)
    empty = dict(empty, keypts_ref=empty["keypts_ref"][:0], bearings_ref=empty["bearings_ref"][:0], ref_matches_with_cur=empty["ref_matches_with_cur"][:0])
    ps.append(empty)
    ps += [IP.problem(10, seed=4), IP.problem(250, scene="planar", seed=5), IP.problem(2000, noise=0.5, seed=6)]
    seeds = [0] * 6 + list(range(100, 94 + len(ps)))   # the status problems with test_every_status's seed
    batch = _gpu(lib_init, ps, True, seeds)
    again = _gpu(lib_init, ps, True, seeds)
    for p, g, a, s in zip(ps, batch, again, seeds):
        single = _gpu(lib_init, [p], True, [s])[0]
        for k in g:
            if isinstance(g[k], np.ndarray):
                assert np.array_equal(g[k], single[k]) and np.array_equal(g[k], a[k]), k
            else:
                assert g[k] == single[k] == a[k], k
        _assert_equal(p, g, _oracle(p, s))
    assert {g["status"] for g in batch} >= {"ok", "no valid model", "decomposition refused", "too few", "ambiguous", "small parallax"}
    assert {g["model"] for g in batch} >= {"H", "F"}


def test_solvers_equal_the_standalone_entries(lib_init):
    from openvslam_b200 import solve
    ps = [IP.problem(400, scene="planar", wrong=0.2, noise=1.0, seed=1), IP.problem(600, wrong=0.3, noise=1.0, seed=2)]
    seeds = [7, 8]
    got = _gpu(lib_init, ps, True, seeds)
    es = [IP.problem(500, camera="equirect", wrong=0.2, noise=1.0, seed=3)]
    got_e = _gpu(lib_init, es, False, [9])
    for s, (cls, key) in enumerate([(solve.homography_solver, "H_21"), (solve.fundamental_solver, "F_21")]):
        h = cls()
        try:
            probs = []
            for p in ps:
                ri = np.nonzero(p["ref_matches_with_cur"] >= 0)[0]
                probs.append(dict(keypts_1=p["keypts_ref"], keypts_2=p["keypts_cur"], matches_12=np.stack([ri, p["ref_matches_with_cur"][ri]], 1)))
            ref = h.find_via_ransac(probs, 100, True, seeds)
        finally:
            h.close()
        for g, r in zip(got, ref):
            assert np.array_equal(g["solver_M"][s], r[key]) and g["solver_score"][s] == r["best_score"]
            assert g["solver_num_inliers"][s] == r["num_inliers"] and g["solver_valid"][s] == r["valid"]
    h = solve.essential_solver()
    try:
        p = es[0]
        ri = np.nonzero(p["ref_matches_with_cur"] >= 0)[0]
        r = h.find_via_ransac([dict(bearings_1=p["bearings_ref"][ri], bearings_2=p["bearings_cur"][p["ref_matches_with_cur"][ri]])], 100, True, [9])[0]
    finally:
        h.close()
    g = got_e[0]
    assert np.array_equal(g["solver_M"][0], r["E_21"]) and g["solver_score"][0] == r["best_score"]
    assert g["solver_num_inliers"][0] == r["num_inliers"] and g["solver_valid"][0] == r["valid"]


@pytest.mark.parametrize("B", [1, 2, 20])
def test_launch_counts(lib_init, B):
    from openvslam_b200 import _lib
    kinds = {"H": [IP.problem(150, scene="planar", seed=s) for s in (1, 3, 4)], "F": [IP.problem(150, seed=s) for s in range(3)]}
    mixed = [kinds["H"][0], kinds["F"][0], IP.problem(5, seed=9), kinds["H"][1], kinds["F"][1], kinds["H"][2], kinds["F"][2]]
    for name, pool in [("all-H", kinds["H"]), ("all-F", kinds["F"]), ("mixed", mixed)]:
        ps = [pool[k % len(pool)] for k in range(B)]
        models = {"all-H": {"H"}, "all-F": {"F"}, "mixed": [{"H"}, {"H", "F"}, {"H", "F", None}][min(B, 3) - 1]}[name]
        for iters, expect in ((100, 13), (0, 7)):
            before = _lib.launch_count()
            got = _gpu(lib_init, ps, True, num_ransac_iters=iters)
            assert _lib.launch_count() - before == expect, (name, iters)
            if iters:
                seen = {g["model"] for g in got}
                assert seen == models, (name, seen)
    es = [IP.problem(150, camera="equirect", seed=k % 3) for k in range(B)]
    for iters, expect in ((100, 8), (0, 6)):
        before = _lib.launch_count()
        _gpu(lib_init, es, False, num_ransac_iters=iters)
        assert _lib.launch_count() - before == expect
    # no match at all, and B == 0: no launch
    p = IP.problem(50, seed=1)
    none = dict(p, ref_matches_with_cur=-np.ones_like(p["ref_matches_with_cur"]))
    before = _lib.launch_count()
    g = _gpu(lib_init, [none] * B, True)
    assert _lib.launch_count() == before and all(x["status"] == "no valid model" and not x["is_triangulated"].any() for x in g)
    assert _gpu(lib_init, [], True) == [] and _lib.launch_count() == before


def test_bad_arguments_launch_nothing(lib_init):
    from openvslam_b200 import _lib
    initialize, optimize = lib_init
    p = IP.problem(100, seed=1)
    e = IP.problem(100, camera="equirect", seed=1)
    bad = []
    q = dict(p, ref_matches_with_cur=p["ref_matches_with_cur"].copy()); q["ref_matches_with_cur"][0] = len(q["keypts_cur"]); bad.append((q, True, {}))
    q = dict(p, ref_matches_with_cur=p["ref_matches_with_cur"].copy()); q["ref_matches_with_cur"][0] = -2; bad.append((q, True, {}))
    q = dict(p, bearings_ref=p["bearings_ref"] * 1.01); bad.append((q, True, {}))
    q = dict(p, keypts_cur=p["keypts_cur"].copy()); q["keypts_cur"][3, 0] = np.nan; bad.append((q, True, {}))
    bad.append((e, True, {}))                      # an equirectangular camera on the perspective initialiser
    bad.append((p, False, {}))                     # a perspective camera on the bearing-vector initialiser
    bad.append((p, True, dict(parallax_deg_thr=float("nan"))))
    bad.append((p, True, dict(parallax_deg_thr=-1.0)))
    bad.append((p, True, dict(reproj_err_thr_sq=float("inf"))))
    bad.append((p, True, dict(num_ransac_iters=-1)))
    bad.append((p, True, dict(min_num_triangulated=-1)))
    for q, persp, kw in bad:
        before = _lib.launch_count()
        with pytest.raises(_lib.OvsError) as ei:
            _gpu(lib_init, [IP.problem(60, seed=2), q], persp, **kw)
        assert ei.value.code == -1 and _lib.launch_count() == before


def test_shared_handle_entries_unchanged(lib_init):
    """brute-force, essential, homography, fundamental, triangulator and create_new_landmarks entries give the same results on a
    handle that also runs initialiser calls"""
    from openvslam_b200 import initialize, match, module, solve
    import triangulation_problems as TP
    rng = np.random.default_rng(0)
    d1 = rng.integers(0, 256, (300, 32), dtype=np.uint8); d2 = d1.copy(); d2[::3, :4] ^= 0xff
    p = IP.problem(300, seed=1)
    ri = np.nonzero(p["ref_matches_with_cur"] >= 0)[0]
    tv = dict(keypts_1=p["keypts_ref"], keypts_2=p["keypts_cur"], matches_12=np.stack([ri, p["ref_matches_with_cur"][ri]], 1))
    ev = dict(bearings_1=p["bearings_ref"][ri], bearings_2=p["bearings_cur"][p["ref_matches_with_cur"][ri]])
    init = initialize.perspective(None)
    users = dict(bf=match.robust(lowe_ratio=0.75), es=solve.essential_solver(), hs=solve.homography_solver(), fs=solve.fundamental_solver(),
                 tv=module.two_view_triangulator(1.0))
    tri = TP.pair_problem(5, 500)
    kf1, nbs, E, ep = TP.neighbourhood(6, 1500, 3)
    own = {k: u._h for k, u in users.items()}
    try:
        for u in users.values():
            u._h = init._h

        def run_all():
            out = [users["bf"].brute_force_match(d1, d2), users["es"].find_via_ransac([ev], 50, True, [1])[0],
                   users["hs"].find_via_ransac([tv], 50, True, [2])[0], users["fs"].find_via_ransac([tv], 50, True, [3])[0]]
            (v, pos), = users["tv"].triangulate([tri])
            rec, rpos = module.create_new_landmarks(users["tv"], kf1, nbs, E, ep, True)
            out += [dict(valid=v, pos=pos), dict(rec=rec, pos=rpos)]
            return out
        first = run_all()
        init.initialize_batch([dict(ref=_view(initialize, lib_init[1], p, "ref"), cur=_view(initialize, lib_init[1], p, "cur"),
                                    ref_matches_with_cur=p["ref_matches_with_cur"])] * 3)
        second = run_all()
        for a, b in zip(first, second):
            if isinstance(a, dict):
                for k in a:
                    assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
            else:
                assert np.array_equal(a, b)
    finally:
        for k, u in users.items():
            u._h = own[k]
            u.close()
        init.close()


def test_cpp_initializer(tmp_path):
    """the class layer and the data::frame adapter (tests/cpp/test_initializer.cpp) on the GPU"""
    import os
    import subprocess
    from openvslam_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build.build()
    libdir = os.path.join(root, "openvslam_b200", "lib")
    exe = str(tmp_path / "test_initializer")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "tests", "cpp", "standin"),
                           os.path.join(root, "tests", "cpp", "test_initializer.cpp"), "-L", libdir, "-lovs_b200", "-Wl,-rpath," + libdir,
                           "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "perspective ok" in r.stdout and "bearing_vector ok" in r.stdout
