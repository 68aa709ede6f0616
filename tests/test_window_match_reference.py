"""The oracle's windowed matchers (oracle/match_oracle.c: projection match_frame_and_landmarks, the match_best loop behind
current_and_last / frame_and_keyframe / Sim3, area match_in_consistent_area, angle_checker, get_keypoints_in_cell) against
the sequential numpy restatement in window_match_reference.py, on the named cases.  Every case also asserts that it
reaches the edges it is named for.  No GPU: this pins the oracle that the GPU parity tests trust."""
import numpy as np
import pytest

import window_match_reference as R


def check_expectations(case, stats):
    for call, name, minimum in case.expect:
        assert stats[call][name] >= minimum, (case.name, call, case.calls[call][0], name, stats[call][name], minimum)


def assert_same(case, i, kind, got, want):
    """got: a matcher's result tuple; want: the reference's (its last item is the stats)."""
    what = "%s call %d (%s)" % (case.name, i, kind)
    if kind == "topk":
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), what
    elif kind == "angles":
        assert np.array_equal(got[0], want[0]), what
    else:
        assert got[0] == want[0], (what, got[0], want[0])
        assert np.array_equal(got[1], want[1]), (what, np.flatnonzero(got[1] != want[1])[:10])
        if kind == "area":
            assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32)), what


def run_case(oracle, case):
    stats = []
    for i, (kind, kw) in enumerate(case.calls):
        want = R.run_reference(case, kind, kw)
        assert_same(case, i, kind, R.run_oracle(oracle, case, kind, kw), want)
        stats.append(want[-1])
    check_expectations(case, stats)


@pytest.mark.parametrize("name", sorted(R.SYNTHETIC_CASES))
def test_oracle_matches_reference(oracle, name):
    run_case(oracle, R.SYNTHETIC_CASES[name]())


def _extract(oracle, img, n):
    kps, desc, _ = oracle.extract(img, oracle.params(n))
    return kps, desc


def test_oracle_matches_reference_bench4(oracle):
    from openvslam_b200 import synth
    kps, desc = _extract(oracle, synth.frame(1920, 960, seed=400), 4000)
    assert len(kps) >= 3900
    run_case(oracle, R.bench4(kps, desc))


def test_oracle_matches_reference_bench2(oracle):
    from openvslam_b200 import synth
    a = synth.frame(752, 480, seed=200)
    ka, da = _extract(oracle, a, 1000)
    kb, db = _extract(oracle, synth.shifted(a, 3, 0), 1000)
    run_case(oracle, R.bench2(ka, da, kb, db))


def test_angle_bins_at_rounding_edges():
    """lrintf rounds the exact float halves 15/30, 135/30, 255/30 to the even bins; 45/30 is just above 1.5 in float;
    -0.0 stays in bin 0; -1e-6 + 360.0 rounds to 360.0f, which the second wrap takes back to 0."""
    d = np.array([15.0, 135.0, 255.0, 45.0, -0.0, -1e-6, 359.99997, 345.0], np.float32)
    assert (d * np.float32(np.float32(1) / np.float32(30)))[:3].tolist() == [0.5, 4.5, 8.5]
    assert R.angle_bins(d).tolist() == [0, 4, 8, 2, 0, 0, 12, 12]
