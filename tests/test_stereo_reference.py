"""The stereo oracle (oracle/match_oracle.c: om_stereo_compute) against the independent numpy restatement of
tests/stereo_reference.py, bit for bit, on the scenes of tests/stereo_cases.py; the branches those scenes reach; the
float32 results against a float64 evaluation; and the sub-pixel disparities against the ground truth of a slanted plane."""
import collections

import numpy as np
import pytest

import stereo_cases as SC
import stereo_reference as SR

CASES = SC.all_cases()


@pytest.fixture(scope="module")
def runs(oracle):
    P = oracle.params(2000)
    sf = SC.scale_factors()
    pyr, out = {}, {}
    for c in CASES:
        k = SC.scene_key(c)
        if k not in pyr:
            left, right = SC.images(c)
            pyr[k] = (oracle.build_pyramid(left, P), oracle.build_pyramid(right, P))
        lp, rp = pyr[k]
        o = oracle.stereo_compute(lp, rp, sf, c["kl"], c["dl"], c["kr"], c["dr"], c["fxb"], c["baseline"])
        r = SR.compute(lp, rp, sf, c["kl"], c["dl"], c["kr"], c["dr"], c["fxb"], c["baseline"])
        out[c["name"]] = (c, o, r)
    return out


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_oracle_equals_reference(runs, name):
    c, (xr, dp, n), r = runs[name]
    assert n == r["num_matched"]
    assert np.array_equal(_bits(xr), _bits(r["x_right"])) and np.array_equal(_bits(dp), _bits(r["depth"]))
    reached = {SR.REASONS[k] for k in r["reason"]}
    assert c["expect"] <= reached, (c["expect"] - reached)


def test_every_reason_is_reached(runs):
    counts = collections.Counter(SR.REASONS[k] for _, _, r in runs.values() for k in r["reason"])
    assert set(counts) == set(SR.REASONS), set(SR.REASONS) - set(counts)


def test_median_cases_reach_their_sads(runs):
    """The median cases' SADs are what they were built to be: at exactly 2 x the median, equal on both sides of it."""
    for c, _, r in runs.values():
        if "sads" in c:
            assert sorted(r["sad"][r["sad"] >= 0].tolist()) == c["sads"], c["name"]
            med = c["sads"][len(c["sads"]) // 2]
            rejected = r["reason"] == SR.R["median_rejected"]
            assert np.array_equal(rejected, r["sad"] >= 2 * med), c["name"]
            assert (r["sad"] == 2 * med).any(), c["name"]


def test_identical_pair_rejects_every_match(runs):
    """The reference's behaviour on a noise-free pair: the median SAD is 0, so every match (SAD >= 0) is rejected."""
    _, (xr, _, n), r = runs["identical_pair"]
    assert n > 200 and (xr == -1).all() and (r["sad"][r["reason"] == SR.R["median_rejected"]] == 0).all()


def test_non_finite_keypoints_come_back_unmatched(runs):
    c, (xr, dp, _), r = runs["non_finite"]
    bad = ~(np.isfinite(c["kl"]["x"]) & np.isfinite(c["kl"]["y"]) & (np.abs(c["kl"]["x"]) < SC.COLS) & (np.abs(c["kl"]["y"]) < SC.ROWS))
    assert bad.sum() >= 21 and (xr[bad] == -1).all() and (dp[bad] == -1).all()
    # a right keypoint with a bad coordinate is no candidate: the true match behind it is taken
    assert (r["reason"][~bad] == SR.R["matched"]).sum() >= 12


def _ulps(a32, b64):
    a = np.asarray(a32, np.float32)
    return np.abs(a.astype(np.float64) - b64) / np.spacing(np.abs(a))


def test_float32_results_within_two_ulps_of_float64(runs):
    total = 0
    for c, _, r in runs.values():
        ok = r["x_right"] >= 0
        if not ok.any():
            continue
        total += ok.sum()
        assert _ulps(r["x_right"][ok], r["x_right64"][ok]).max() <= 2, c["name"]
        assert _ulps(r["depth"][ok], r["depth64"][ok]).max() <= 2, c["name"]
    assert total > 2000


def test_subpixel_disparity_against_the_plane(runs):
    """Disparities of the slanted plane d = 20 + 0.02 x (bilinear resampling, noise in [-2, 2]) against the truth.  Measured
    with the oracle (equal to the kernel bit for bit): 1197 matches, |error| median 0.43 px, 90th percentile 0.98 px, 95th
    1.18 px, 99th 1.79 px, one mismatch of 12.1 px; the fractional parts of the disparities fill [0, 1) evenly."""
    c, (xr, _, _), _ = runs["plane"]
    ok = xr >= 0
    x = c["kl"]["x"][ok].astype(np.float64)
    disp = x - xr[ok]
    err = np.abs(disp - (SC.PLANE_D0 + SC.PLANE_A * x))
    assert ok.sum() > 1000
    assert np.median(err) < 0.5 and np.percentile(err, 95) < 1.25 and np.mean(err > 3) < 0.005
    hist = np.histogram(disp % 1.0, bins=10, range=(0, 1))[0]
    assert hist.min() > 0.5 * hist.mean()
