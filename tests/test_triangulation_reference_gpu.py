"""GPU tests of module::two_view_triangulator (k_two_view_triangulate) and of create_new_landmarks' compute step against the
numpy reference tests/triangulation_reference.py, on the constructed cases of tests/triangulation_cases.py: valid flags
(and records) equal, no decision left to the two-camera point's bound on the knife-edge cases, points bit for bit on a
stereo branch and within the bound on the two-camera branch -- and still bit for bit with the oracle."""
import collections

import numpy as np
import pytest

import triangulation_cases as TC
import triangulation_problems as TP
import triangulation_reference as R
from openvslam_b200 import match, module
from test_triangulation_reference import GROUPS, far_stereo_measurement

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def OT(oracle):
    from oracle import triangulation
    return triangulation


@pytest.fixture(scope="module")
def cases():
    by = collections.defaultdict(list)
    for c in TC.knife_edge_cases() + [TC.far_stereo()] + TC.sizes():
        by[c.group].append(c)
    return by


def device_triangulate(problems):
    """one device call per threshold, each a batch of that threshold's problems, in the order given"""
    out = [None] * len(problems)
    for deg in sorted({p[3] for p in problems}):
        idx = [k for k, p in enumerate(problems) if p[3] == deg]
        tv = module.two_view_triangulator(deg)
        for k, got in zip(idx, tv.triangulate([problems[k][:3] for k in idx])):
            out[k] = got
        tv.close()
    return out


@pytest.mark.parametrize("group", GROUPS)
def test_device_matches_the_reference_on_named_cases(OT, cases, group):
    n = collections.Counter()
    for case in cases[group]:
        for (kf1, kf2, pairs, deg), (valid, pos) in zip(case.problems, device_triangulate(case.problems)):
            ref = R.triangulate(kf1, kf2, pairs, deg)
            if case.knife_edge:
                assert not ref.skip, (case.name, ref.skip)
            open_ = np.zeros(len(pairs), bool)
            open_[[k for k, _ in ref.skip]] = True
            assert np.array_equal(valid[~open_], ref.valid[~open_]), (case.name, np.flatnonzero(valid != ref.valid))
            for k in np.flatnonzero(valid & ref.valid):
                if ref.branch[k] == R.TWO_CAMERAS:
                    assert np.linalg.norm(pos[k] - ref.pos[k]) <= ref.bound[k], (case.name, k)
                else:
                    assert pos[k].tobytes() == ref.pos[k].tobytes(), (case.name, k, ref.branch[k])
            ov, opos, _, _ = OT.triangulate(kf1, kf2, pairs, deg)
            assert np.array_equal(valid, ov) and pos.tobytes() == np.ascontiguousarray(opos).tobytes(), case.name
            n["pairs"] += len(pairs); n["valid"] += int(valid.sum()); n["skips"] += len(ref.skip)
    print(group, dict(n))


def test_far_stereo_measurement_on_the_device(cases):
    def points(kf1, kf2, pairs):
        # rays_parallax_deg_thr only matters for two monocular keypoints; every keypoint here is stereo
        (valid, pos), = module.two_view_triangulator(1.0).triangulate([(kf1, kf2, pairs)])
        assert valid.all()
        return pos
    case = cases["far_stereo"][0]
    (kf1, kf2, pairs, deg), = case.problems
    ref = R.triangulate(kf1, kf2, pairs, deg)
    keep = np.flatnonzero(ref.valid)
    sub = TC.Case(case.name, case.group, [(kf1, kf2, pairs[keep], deg)], (), False)
    m = far_stereo_measurement(sub, points)
    print("far stereo (device, valid pairs): %s" % m)
    assert m["worst error / bound"] <= 1.0


# ------------------------------------------------------------------------------------------------ create_new_landmarks


def _same(got, ref, oracle_rec):
    rec, pos, pairs = ref[0], ref[1], ref[2]
    assert np.array_equal(got[0], rec), (len(got[0]), len(rec))
    assert R.same_points(got[1], pairs)
    assert np.array_equal(got[0], oracle_rec[0]) and got[1].tobytes() == np.ascontiguousarray(oracle_rec[1]).tobytes()


@pytest.mark.parametrize("B,check", [(1, False), (2, True), (20, False), (20, True)])
def test_create_new_landmarks_matches_the_reference(OT, B, check):
    kf1, nbs, E, ep = TP.neighbourhood(700 + B, 1500, B, stereo_frac=0.3)
    mt = match.robust(check_orientation=check)
    got = module.create_new_landmarks(mt, kf1, nbs, E, ep, check)
    ref = R.create_new_landmarks(kf1, nbs, E, ep, check)
    _same(got, ref, OT.create_new_landmarks(kf1, nbs, E, ep, check))
    assert len(ref[0]) > 100
    mt.close()


def test_requeried_lists_match_the_reference(OT):
    kf1, nbs, E, ep = TC.planar_neighbourhood(8, 600, 3)
    mt = match.robust(check_orientation=False)
    before = mt.num_requeries()
    got = module.create_new_landmarks(mt, kf1, nbs, E, ep, False)
    ref = R.create_new_landmarks(kf1, nbs, E, ep, False)
    assert mt.num_requeries() > before and ref[3] > 0
    _same(got, ref, OT.create_new_landmarks(kf1, nbs, E, ep, False))
    mt.close()


def test_uneven_neighbours_match_the_reference(OT):
    """neighbours with all, none, a few dozen, half and a few hundred unlisted keypoints: each neighbour's candidates start at
    its own offset of the batched lists"""
    kf1, nbs, E, ep = TC.uneven_neighbourhood(40)
    mt = match.robust(check_orientation=True)
    got = module.create_new_landmarks(mt, kf1, nbs, E, ep, True)
    ref = R.create_new_landmarks(kf1, nbs, E, ep, True)
    _same(got, ref, OT.create_new_landmarks(kf1, nbs, E, ep, True))
    assert set(ref[0][:, 0].tolist()) >= {0, 2, 3, 4} and 1 not in ref[0][:, 0]
    mt.close()


def test_a_neighbour_whose_every_pair_fails_and_the_landmark_carry(OT):
    """neighbour 1 is turned around after its E_12 was formed: its lists are those of the true pose, but every pair it
    matches is behind it.  The neighbours see the same points, so keyframe-1 keypoints that got a landmark from an earlier
    neighbour must drop out of the later neighbours' queries"""
    kf1, nbs, E, ep = TP.neighbourhood(77, 1500, 4, stereo_frac=0.0)
    n = nbs[1]
    Rb = n.pose_cw[:9].reshape(3, 3)
    c = -(Rb.T @ n.pose_cw[9:])
    Rt = TC.R_Y180 @ Rb
    nbs[1] = module.keyframe(np.concatenate([Rt.reshape(9), -Rt @ c]), n.camera, n.scale_factor, n.scale_factors, n.level_sigma_sq,
                             n.keypts["x"], n.keypts["y"], n.keypts["octave"], n.bearings, angle=n.keypts["angle"],
                             true_baseline=n.true_baseline, descriptors=n.descriptors, has_landmark=n.has_landmark, bow_node=n.bow_node)
    mt = match.robust(check_orientation=False)
    got = module.create_new_landmarks(mt, kf1, nbs, E, ep, False)
    ref = R.create_new_landmarks(kf1, nbs, E, ep, False)
    _same(got, ref, OT.create_new_landmarks(kf1, nbs, E, ep, False))
    assert 1 not in ref[0][:, 0] and {0, 2, 3} <= set(ref[0][:, 0].tolist())
    # without the carry a keyframe-1 keypoint would get a landmark from several neighbours
    alone = np.concatenate([R.create_new_landmarks(kf1, [nb], E[b:b + 1], ep[b:b + 1], False)[0][:, 1] for b, nb in enumerate(nbs)])
    assert len(alone) > len(np.unique(alone)) and len(np.unique(got[0][:, 1])) == len(got[0])
    mt.close()
