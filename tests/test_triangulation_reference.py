"""CPU tests of tests/triangulation_reference.py, the numpy reference of the two-view triangulator and of
create_new_landmarks' compute step: against the oracle (oracle/triangulation_oracle.c) and against the device arithmetic
(openvslam_b200/csrc/triangulation_math.cuh through tests/triangulationcheck), on the constructed knife-edge cases of
tests/triangulation_cases.py and on the random scenes of tests/triangulation_problems.py."""
import collections
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import triangulation_cases as TC
import triangulation_problems as TP
import triangulation_reference as R
from test_two_view_triangulator_oracle import _cases as random_cases

HERE = os.path.dirname(os.path.abspath(__file__))
GROUPS = ("parallax", "stereo_parallax", "reprojection", "scale", "cheirality", "far_stereo", "sizes")
GATES = ("parallax", "stereo parallax", "cheirality 1", "cheirality 2", "reprojection 1 mono", "reprojection 1 stereo",
         "reprojection 2 mono", "reprojection 2 stereo", "scale low", "scale high")


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


def oracle_point(kf1, kf2, i1, i2, cos_thr):
    """the oracle's point and branch of one pair whatever its gates decide"""
    import oracle.triangulation as T
    keep = []
    k1 = T._kf(kf1, keep); k2 = T._kf(kf2, keep)
    p = (C.c_double * 3)(); br = C.c_int(0)
    T.lib().otr_triangulate(C.byref(k1), C.byref(k2), int(i1), int(i2), C.c_double(cos_thr), p, C.byref(br))
    return np.array(list(p)), br.value


def check_points(ref, pos, branch, where):
    """pos (m, 3) at the pairs `where`: bit for bit on a stereo branch, within the bound on the two-camera branch"""
    for k in np.flatnonzero(where):
        if branch[k] == R.TWO_CAMERAS:
            if ref.reason[k] != R.NON_FINITE:
                assert np.linalg.norm(pos[k] - ref.pos[k]) <= ref.bound[k], (k, pos[k], ref.pos[k], ref.bound[k])
        elif branch[k] != R.NONE:
            assert pos[k].tobytes() == ref.pos[k].tobytes(), (k, pos[k], ref.pos[k])


def agree(ref, reason, branch, knife_edge):
    """reason and branch equal outside the skips; no skips on a knife-edge case"""
    if knife_edge:
        assert not ref.skip, ref.skip
    skipped = np.zeros(len(ref.reason), bool)
    skipped[[k for k, _ in ref.skip]] = True
    bad = np.flatnonzero(((ref.reason != reason) | (ref.branch != branch)) & ~skipped)
    assert len(bad) == 0, [(int(k), int(ref.reason[k]), int(reason[k]), int(ref.branch[k]), int(branch[k])) for k in bad[:10]]


@pytest.mark.parametrize("group", GROUPS)
def test_reference_matches_the_oracle_on_named_cases(OT, cases, group):
    seen = collections.Counter()
    for case in cases[group]:
        counts = collections.Counter()
        for kf1, kf2, pairs, deg in case.problems:
            ref = R.triangulate(kf1, kf2, pairs, deg)
            valid, pos, reason, branch = OT.triangulate(kf1, kf2, pairs, deg)
            agree(ref, reason, branch, case.knife_edge)
            raw = np.array([oracle_point(kf1, kf2, i1, i2, R.cos_threshold(deg))[0] for i1, i2 in pairs]).reshape(-1, 3)
            check_points(ref, raw, branch, np.ones(len(pairs), bool))
            assert np.array_equal(valid, ref.valid)
            counts.update(ref.gates)
        for want in case.expect:
            assert counts[want] > 0, (case.name, want, counts)
        seen.update(counts)
    print(group, dict(sorted(seen.items(), key=str)))


def test_every_gate_is_reached_with_both_outcomes(cases):
    """over the constructed cases (not the random far_stereo and sizes scenes)"""
    seen = collections.Counter()
    for group in ("parallax", "stereo_parallax", "reprojection", "scale", "cheirality"):
        for case in cases[group]:
            for kf1, kf2, pairs, deg in case.problems:
                seen.update(R.triangulate(kf1, kf2, pairs, deg).gates)
    print(dict(sorted(seen.items(), key=str)))
    for g in GATES:
        assert seen[(g, True)] > 0 and seen[(g, False)] > 0, g
    for b in R.BRANCHES.values():
        assert seen[("branch", b)] > 0, b


def test_reference_matches_the_oracle_on_random_scenes(OT):
    skips = 0
    for kf1, kf2, pairs in random_cases():
        ref = R.triangulate(kf1, kf2, pairs)
        valid, pos, reason, branch = OT.triangulate(kf1, kf2, pairs)
        agree(ref, reason, branch, False)
        check_points(ref, pos, branch, valid)
        skips += len(ref.skip)
    print("random scenes: %d decisions left to the bound" % skips)
    assert skips == 0


def test_far_stereo_measurement(OT, cases):
    """the oracle's Jacobi point (the device's bits) against the SVD point at 0.06 - 0.6 degrees of parallax"""
    m = far_stereo_measurement(cases["far_stereo"][0], lambda kf1, kf2, pairs: [oracle_point(kf1, kf2, i1, i2, R.cos_threshold(1.0))[0]
                                                                               for i1, i2 in pairs])
    print("far stereo (oracle): %s" % m)
    assert m["two-camera pairs"] > 300 and m["worst error / bound"] <= 1.0


def far_stereo_measurement(case, points):
    """worst |point - SVD point| (absolute, relative), its ratio to the bound, and how many gate decisions the bound leaves
    open, over the two-camera pairs of the far_stereo case; points(kf1, kf2, pairs) -> the points to measure"""
    (kf1, kf2, pairs, deg), = case.problems
    ref = R.triangulate(kf1, kf2, pairs, deg)
    two = np.flatnonzero((ref.branch == R.TWO_CAMERAS) & (ref.reason != R.NON_FINITE))
    got = np.array(points(kf1, kf2, pairs[two])).reshape(-1, 3)
    err = np.linalg.norm(got - ref.pos[two], axis=1)
    par = [math.degrees(math.acos(min(1.0, ref.pairs[k].cos_rays))) for k in two]
    return {"two-camera pairs": int(len(two)), "parallax deg": (round(min(par), 3), round(max(par), 3)),
            "worst error m": float(err.max()), "worst relative error": float((err / np.linalg.norm(ref.pos[two], axis=1)).max()),
            "worst error / bound": float((err / ref.bound[two]).max()), "decisions inside the bound": len(ref.skip),
            "gates open": sorted(collections.Counter(g for _, g in ref.skip).items())}


@pytest.fixture(scope="module")
def triangulationcheck(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("triangulationcheck") / "libtriangulationcheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-x", "c++", "-shared", "-o", so,
                           os.path.join(HERE, "triangulationcheck", "triangulationcheck.cpp"), "-lm"])
    return C.CDLL(so)


def header_triangulate(lib, kf1, kf2, pairs, deg):
    """triangulation_math.cuh's tri_two_view over the pairs -> reason, branch, pos (zero where invalid)"""
    keep = []
    k1, k2 = kf1.view(), kf2.view()
    keep += [k1, k2]
    m = len(pairs)
    pos = np.zeros((max(m, 1), 3)); reason = np.zeros(max(m, 1), np.int32); branch = np.zeros(max(m, 1), np.int32)
    pr = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib.tc_two_view_triangulate(C.byref(k1), C.byref(k2), m, vp(pr), C.c_double(R.cos_threshold(deg)), vp(pos), vp(reason), vp(branch))
    return reason[:m], branch[:m], pos[:m]


@pytest.mark.parametrize("group", GROUPS)
def test_header_matches_the_reference(triangulationcheck, cases, group):
    for case in cases[group]:
        for kf1, kf2, pairs, deg in case.problems:
            ref = R.triangulate(kf1, kf2, pairs, deg)
            reason, branch, pos = header_triangulate(triangulationcheck, kf1, kf2, pairs, deg)
            agree(ref, reason, branch, case.knife_edge)
            check_points(ref, pos, branch, reason == R.OK)


def test_header_matches_the_reference_on_random_scenes(triangulationcheck):
    for kf1, kf2, pairs in random_cases():
        ref = R.triangulate(kf1, kf2, pairs)
        reason, branch, pos = header_triangulate(triangulationcheck, kf1, kf2, pairs, 1.0)
        agree(ref, reason, branch, False)
        check_points(ref, pos, branch, reason == R.OK)


def test_stereo_parallax_forms_differ_by_a_few_ulp():
    """(d^2 - h^2) / (d^2 + h^2) against the recalled cos(2 atan2(h, d)), over depths 0.05 - 1000 m and baselines 0.05 - 1 m:
    they differ by at most a couple of ulp of 1 (relative to the value, by hundreds of ulp where it is near 0, d near h).
    cos_rays is compared with them, so that is how close to a stereo-parallax decision the two forms can disagree."""
    worst = 0.0
    for tb in (0.05, 0.12, 0.3, 0.5, 1.0):
        for d in np.geomspace(0.05, 1000.0, 2000).astype(np.float32):
            kf = TC.View(np.eye(3), [0, 0, 0], true_baseline=tb)
            kf.add([0.0, 0.0, 1.0], TC.CX, TC.CY, 0, 1.0, d)
            k = kf.keyframe()
            worst = max(worst, abs(R.stereo_cos(k, 0) - R.stereo_cos_atan2(k, 0)) / R.EPS)
    print("closed form against cos(2 atan2(h, d)): %.1f eps at most" % worst)
    assert worst <= 2.0


# ------------------------------------------------------------------------------------------------ create_new_landmarks


def check_records(ref, got):
    """records equal; points: bit for bit on a stereo branch, within the bound on the two-camera branch"""
    rec, pos, pairs = ref[0], ref[1], ref[2]
    assert np.array_equal(got[0], rec), (len(got[0]), len(rec))
    assert R.same_points(got[1], pairs)


NEIGHBOURHOODS = {"B1": lambda: TP.neighbourhood(21, 1500, 1, stereo_frac=0.3), "B6": lambda: TP.neighbourhood(26, 1500, 6, stereo_frac=0.3),
                  "B12": lambda: TP.neighbourhood(32, 1500, 12, stereo_frac=0.3), "planar": lambda: TC.planar_neighbourhood(8, 600, 3),
                  "uneven": lambda: TC.uneven_neighbourhood(40)}


@pytest.mark.parametrize("check", [False, True])
@pytest.mark.parametrize("name", sorted(NEIGHBOURHOODS))
def test_reference_create_new_landmarks_matches_the_oracle(OT, name, check):
    kf1, nbs, E, ep = NEIGHBOURHOODS[name]()
    ref = R.create_new_landmarks(kf1, nbs, E, ep, check)
    check_records(ref, OT.create_new_landmarks(kf1, nbs, E, ep, check))
    assert len(ref[0]) > 20
    if name == "planar":
        assert ref[3] > 0                      # the lists ran out: re-queried
    if name == "uneven":
        assert set(ref[0][:, 0].tolist()) >= {0, 2, 3, 4} and 1 not in ref[0][:, 0]
