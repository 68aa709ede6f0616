"""GPU tests of module::two_view_triangulator (ovs_two_view_triangulate_host) and of create_new_landmarks' compute step
(ovs_create_new_landmarks_host) against the oracle: valid flags and records identical, points bit for bit."""
import ctypes as C

import numpy as np
import pytest

import triangulation_problems as TP
from triangulation_cases import planar_neighbourhood as _planar_neighbourhood
from openvslam_b200 import _lib, match, module

pytestmark = pytest.mark.gpu

CONFIGS = {"mono": ("perspective", 0.0, 0.4), "stereo": ("perspective", 1.0, 0.4), "mixed": ("perspective", 0.5, 0.05),
           "equirectangular": ("equirectangular", 0.0, 0.4)}


@pytest.fixture(scope="module")
def OT(oracle):
    from oracle import triangulation
    return triangulation


def _problem(cfg, m, seed):
    model, st, sp = CONFIGS[cfg]
    return TP.pair_problem(seed, m, model, st, sp)


def _same(got, ref):
    (v, p), (ov, op) = got, ref[:2]
    assert np.array_equal(v, ov) and p.tobytes() == np.ascontiguousarray(op).tobytes()


@pytest.mark.parametrize("cfg", sorted(CONFIGS))
@pytest.mark.parametrize("m", [1, 31, 32, 33, 255, 256, 257, 4000, 20000])
def test_batched_triangulation_matches_the_oracle(OT, cfg, m):
    kf1, kf2, pairs = _problem(cfg, m, 100 + m)
    tv = module.two_view_triangulator(1.0)
    (got,) = tv.triangulate([(kf1, kf2, pairs)])
    ref = OT.triangulate(kf1, kf2, pairs, 1.0)
    _same(got, ref)
    if m >= 4000:
        assert 0.1 < got[0].mean() < 0.9
    tv.close()


@pytest.mark.parametrize("B", [3, 20])
def test_a_batch_equals_its_single_calls(OT, B):
    rng = np.random.default_rng(B)
    cfgs = sorted(CONFIGS)
    probs = [_problem(cfgs[b % 4], int(rng.integers(0, 700)), 300 + b) for b in range(B)]
    probs[1] = (probs[1][0], probs[1][1], np.zeros((0, 2), np.int32))          # an empty problem inside a batch
    tv = module.two_view_triangulator(1.0)
    batch = tv.triangulate(probs)
    for b, (kf1, kf2, pairs) in enumerate(probs):
        if len(pairs):
            _same(batch[b], tv.triangulate([(kf1, kf2, pairs)])[0])
        _same(batch[b], OT.triangulate(kf1, kf2, pairs, 1.0))
    tv.close()


def test_empty_problems_make_no_launch():
    kf1, kf2, _ = _problem("mono", 10, 1)
    tv = module.two_view_triangulator(1.0)
    before = _lib.launch_count()
    assert tv.triangulate([]) == []
    out = tv.triangulate([(kf1, kf2, np.zeros((0, 2), np.int32))] * 3)
    assert all(len(v) == 0 for v, _ in out)
    assert _lib.launch_count() == before
    tv.close()


def _with(kf, **kw):
    """a copy of keyframe kf with some of its fields replaced"""
    a = dict(pose_cw=kf.pose_cw, camera=kf.camera, scale_factor=kf.scale_factor, scale_factors=kf.scale_factors,
             level_sigma_sq=kf.level_sigma_sq, x=kf.keypts["x"], y=kf.keypts["y"], octave=kf.keypts["octave"].copy(), bearings=kf.bearings.copy(),
             angle=kf.keypts["angle"], stereo_x_right=kf.stereo_x_right, depths=kf.depths, true_baseline=kf.true_baseline,
             descriptors=kf.descriptors, has_landmark=kf.has_landmark, bow_node=kf.bow_node)
    a.update(kw)
    return module.keyframe(**a)


def test_bad_arguments_are_rejected_before_any_launch():
    from openvslam_b200 import optimize
    kf1, kf2, pairs = _problem("mixed", 50, 2)
    st = kf2.stereo_x_right >= 0
    oct_bad = kf1.keypts["octave"].copy(); oct_bad[pairs[3, 0]] = 8
    b_bad = kf2.bearings.copy(); b_bad[pairs[4, 1]] *= 1.01
    d_bad = kf2.depths.copy(); d_bad[np.flatnonzero(st)[0]] = np.nan
    bad = [(kf1, kf2, pairs + np.array([0, kf2.num_keypts], np.int32) * (np.arange(len(pairs))[:, None] == 7)),
           (kf1, kf2, pairs - np.array([1 << 20, 0], np.int32) * (np.arange(len(pairs))[:, None] == 9)),
           (_with(kf1, octave=oct_bad), kf2, pairs),
           (kf1, _with(kf2, bearings=b_bad), pairs),
           (kf1, _with(kf2, depths=d_bad), pairs),
           (kf1, _with(kf2, camera=optimize.camera("fisheye", 500, 500, 320, 240)), pairs),
           (kf1, _with(kf2, camera=optimize.camera("equirectangular", cols=2000, rows=1000)), pairs),     # stereo keypoints
           (_with(kf1, pose_cw=np.full(12, np.nan)), kf2, pairs)]
    tv = module.two_view_triangulator(1.0)
    before = _lib.launch_count()
    for k, prob in enumerate(bad):
        with pytest.raises(_lib.OvsError) as e:
            tv.triangulate([(kf1, kf2, pairs[:5]), prob])
        assert e.value.code == -1, k
    tv.rays_parallax_deg_thr_ = float("nan")
    with pytest.raises(_lib.OvsError):
        tv.triangulate([(kf1, kf2, pairs)])
    rc = _lib.lib().ovs_two_view_triangulate_host(tv._h, 65536, None, None, None, None, C.c_double(1.0), None, None)
    assert rc == -1
    assert _lib.launch_count() == before
    tv.close()


# ------------------------------------------------------------------ create_new_landmarks


def _sequential(OT, kf1, nbs, E, ep, check):
    return OT.create_new_landmarks(kf1, nbs, E, ep, check, 1.0)


def _same_records(got, ref):
    assert np.array_equal(got[0], ref[0]) and got[1].tobytes() == np.ascontiguousarray(ref[1]).tobytes()


@pytest.mark.parametrize("B,n1,check", [(1, 1500, False), (2, 1500, True), (10, 1500, False), (20, 1500, True), (1, 4000, True),
                                        (2, 4000, False), (10, 4000, True), (20, 4000, False)])
def test_create_new_landmarks_matches_the_sequential_loop(OT, B, n1, check):
    kf1, nbs, E, ep = TP.neighbourhood(500 + B + n1, n1, B, stereo_frac=0.3)
    mt = match.robust(check_orientation=check)
    got = module.create_new_landmarks(mt, kf1, nbs, E, ep, check)
    ref = _sequential(OT, kf1, nbs, E, ep, check)
    _same_records(got, ref)
    assert len(got[0]) > 0.1 * n1 and len(set(got[0][:, 0].tolist())) > B // 2
    # the same call again on the same handle gives the same bits
    _same_records(module.create_new_landmarks(mt, kf1, nbs, E, ep, check), got)
    mt.close()


def test_carrying_the_landmark_flags_changes_the_result(OT):
    """neighbours observe the same points: treating them as independent problems would give keyframe-1 keypoints several landmarks"""
    kf1, nbs, E, ep = TP.neighbourhood(7, 1500, 6)
    mt = match.robust(check_orientation=True)
    got = module.create_new_landmarks(mt, kf1, nbs, E, ep, True)
    _same_records(got, _sequential(OT, kf1, nbs, E, ep, True))
    indep = [module.create_new_landmarks(mt, kf1, [n], E[b:b + 1], ep[b:b + 1], True) for b, n in enumerate(nbs)]
    rec = np.concatenate([np.column_stack([np.full(len(r), b), r[:, 1:]]) for b, (r, _) in enumerate(indep)])
    assert len(rec) > len(got[0]) and len(np.unique(got[0][:, 1])) == len(got[0])
    mt.close()


def test_exhausted_lists_are_requeried(OT):
    kf1, nbs, E, ep = _planar_neighbourhood(8, 600, 3)
    mt = match.robust(check_orientation=False)
    before = mt.num_requeries()
    got = module.create_new_landmarks(mt, kf1, nbs, E, ep, False)
    assert mt.num_requeries() > before
    _same_records(got, _sequential(OT, kf1, nbs, E, ep, False))
    mt.close()


def test_prefix_of_the_neighbours_gives_the_prefix_of_the_records(OT):
    kf1, nbs, E, ep = TP.neighbourhood(9, 1500, 10, stereo_frac=0.3)
    mt = match.robust(check_orientation=True)
    rec, pos = module.create_new_landmarks(mt, kf1, nbs, E, ep, True)
    for k in (1, 4, 9):
        keep = rec[:, 0] < k
        prec, ppos = module.create_new_landmarks(mt, kf1, nbs[:k], E[:k], ep[:k], True)
        assert np.array_equal(prec, rec[keep]) and ppos.tobytes() == pos[keep].tobytes()
    mt.close()


def test_launch_count_does_not_depend_on_the_number_of_neighbours():
    kf1, nbs, E, ep = TP.neighbourhood(10, 2000, 20)
    mt = match.robust(check_orientation=False)
    counts = []
    for B in (1, 2, 20):
        rq = mt.num_requeries()
        before = _lib.launch_count()
        rec, _ = module.create_new_landmarks(mt, kf1, nbs[:B], E[:B], ep[:B], False)
        assert mt.num_requeries() == rq and len(rec) > 0
        counts.append(_lib.launch_count() - before)
    assert counts == [3, 3, 3]
    mt.close()


def test_the_triangulation_matcher_is_unchanged_on_a_shared_handle(oracle):
    from openvslam_b200 import synth
    p = synth.triangulation_problem(1500, 1)
    sf = oracle.scale_factors(1.2, 8)
    keys = ("desc_1", "bearing_1", "octave_1", "angle_1", "has_lm_1", "is_stereo_1", "bow_node_1",
            "desc_2", "bearing_2", "angle_2", "has_lm_2", "is_stereo_2", "bow_node_2", "E_12", "epipole_in_2")
    mt = match.robust(check_orientation=True)
    first = mt.match_for_triangulation(*[p[k] for k in keys], sf)
    kf1, nbs, E, ep = TP.neighbourhood(11, 4000, 10)
    module.create_new_landmarks(mt, kf1, nbs, E, ep, True)
    again = mt.match_for_triangulation(*[p[k] for k in keys], sf)
    onum, om = oracle.robust_match_for_triangulation(*[p[k] for k in keys], sf, True)
    assert first[0] == again[0] == onum and np.array_equal(first[1], again[1]) and np.array_equal(again[1], om)
    mt.close()


def test_create_new_landmarks_rejects_bad_arguments_before_any_launch():
    kf1, nbs, E, ep = TP.neighbourhood(12, 500, 3, stereo_frac=0.3)
    mt = match.robust()
    before = _lib.launch_count()
    bad_oct = kf1.keypts["octave"].copy(); bad_oct[5] = -1
    cases = [(_with(kf1, octave=bad_oct), nbs, E, ep), (kf1, nbs[:2] + [_with(nbs[2], descriptors=None)], E, ep),
             (kf1, nbs, np.full_like(E, np.nan), ep)]
    for k1, n, e, p in cases:
        with pytest.raises(_lib.OvsError) as err:
            module.create_new_landmarks(mt, k1, n, e, p)
        assert err.value.code == -1
    assert _lib.launch_count() == before
    mt.close()


def test_create_new_landmarks_rejects_more_candidate_slots_than_a_call_holds():
    """65535 neighbours x 4100 queries x 8 list slots is above 2^31 - 1: refused on the host, nothing launched"""
    kf1, nbs, _, _ = TP.neighbourhood(13, 4400, 1)
    kf1 = _with(kf1, has_landmark=np.zeros(kf1.num_keypts, np.uint8), bow_node=np.zeros(kf1.num_keypts, np.int32))
    n = nbs[0]
    one = module.keyframe(n.pose_cw, n.camera, n.scale_factor, n.scale_factors, n.level_sigma_sq, n.keypts["x"][:1], n.keypts["y"][:1],
                          n.keypts["octave"][:1], n.bearings[:1], descriptors=n.descriptors[:1], has_landmark=np.zeros(1, np.uint8),
                          bow_node=np.zeros(1, np.int32))
    B = 65535
    mt = match.robust()
    before = _lib.launch_count()
    with pytest.raises(_lib.OvsError) as err:
        module.create_new_landmarks(mt, kf1, [one] * B, np.tile(np.eye(3), (B, 1, 1)), np.tile([0.0, 0.0, 1.0], (B, 1)))
    assert err.value.code == -6
    assert _lib.launch_count() == before
    mt.close()


def test_cpp_two_view_triangulator(tmp_path):
    """the class layer and the data::keyframe adapter (tests/cpp/test_two_view_triangulator.cpp) on the GPU"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "openvslam_b200", "lib")
    exe = str(tmp_path / "test_two_view_triangulator")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "tests", "cpp", "standin"),
                           os.path.join(root, "tests", "cpp", "test_two_view_triangulator.cpp"), "-L", libdir, "-lovs_b200",
                           "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "two-view triangulator ok" in r.stdout, r.stdout + r.stderr
