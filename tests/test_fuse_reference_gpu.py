"""match::fuse::replace_duplication on the device (ovs_fuse_replace_duplication_host) and the fuse matching core
(ovs_fuse_best_keypoints_host) against the numpy reference of tests/fuse_reference.py, query by query, on every named case: the
chi-square gate at 5.99f and 7.8f exactly and one float above, keypoint x_right of -1, -0.0, 0.0 and the smallest positive
float, the level range at its edges on 1- to 16-level scale tables, the box edge and clipped windows on irregular grids, the
Hamming acceptance at 50 / 51 and first-visited ties, ranks past 32768 and 65280, a mixed batch and 120 benchmark-sized targets."""
import numpy as np
import pytest

from openvslam_b200 import match
import fuse_reference as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fz():
    m = match.fuse()
    yield m
    m.close()


def device_target(t):
    f, g = t.frame, t.frame.grid
    return match.fuse_target(t.geometry, t.scale_factors, t.inv_level_sigma_sq, f.x, f.y, f.octave, f.desc,
                             match.camera_grid(*g.bounds, g.cols, g.rows), x_right=f.x_right)


def run_device(fz, c, targets=None, q_off=None, q_lm=None):
    targets = c.targets if targets is None else targets
    q_off = c.q_off if q_off is None else q_off
    q_lm = c.q_lm if q_lm is None else q_lm
    L = c.lms
    return fz.replace_duplication([device_target(t) for t in targets], L["pos_w"], L["mean_normal"], L["min_valid_dist"], L["max_valid_dist"],
                                  L["lm_desc"], q_off, q_lm, c.margin, geometry=True)


@pytest.mark.parametrize("name", sorted(R.CASES))
def test_device_equals_reference(fz, name):
    c, ref = R.case_and_reference(name)
    num, best, ok, uv, xr, lv = run_device(fz, c)
    _, rbest, rok, ruv, rxr, rlv, _ = ref
    assert np.array_equal(ok, rok) and np.array_equal(lv, rlv)
    assert xr.tobytes() == rxr.tobytes()
    assert num == int((best >= 0).sum())
    for k, t in enumerate(c.targets):
        s = slice(c.q_off[k], c.q_off[k + 1])
        if not c.equirect[k]:
            assert uv[s].tobytes() == ruv[s].tobytes(), k
            assert np.array_equal(best[s], rbest[s]), (k, np.flatnonzero(best[s] != rbest[s])[:8])
        else:
            # the device's atan2 / asin: at most one float ulp on the reprojection; the search must be the reference's on the
            # device's own reprojection
            ulps = np.abs(uv[s].view(np.int32).astype(np.int64) - ruv[s].view(np.int32).astype(np.int64))
            assert ulps.max(initial=0) <= 1, k
            rows = np.maximum(c.q_lm[s], 0)
            b, _ = R.search(t, ok[s], uv[s], xr[s], lv[s], c.lms["lm_desc"][rows], c.margin)
            assert np.array_equal(best[s], b), k
    if not any(c.equirect):
        assert num == ref[0]


@pytest.mark.parametrize("name", sorted(R.CASES))
def test_best_keypoints_equals_reference(fz, name):
    """ovs_fuse_best_keypoints_host on each target's frame index, fed the reference's reprojections."""
    c, ref = R.case_and_reference(name)
    _, rbest, rok, ruv, rxr, rlv, _ = ref
    checked = 0
    for k, t in enumerate(c.targets):
        s = slice(c.q_off[k], c.q_off[k + 1])
        if s.stop == s.start or t.n == 0:
            continue
        f = t.frame
        idx = match.frame_index(fz, f.x, f.y, f.octave, f.angle, f.x_right, f.desc, match.camera_grid(*f.grid.bounds, f.grid.cols, f.grid.rows))
        try:
            rows = np.maximum(c.q_lm[s], 0)
            n, best = fz.best_keypoints(idx, ruv[s], rxr[s], rlv[s], c.lms["lm_desc"][rows], t.scale_factors, t.inv_level_sigma_sq, c.margin,
                                        usable=rok[s].astype(np.uint8))
        finally:
            idx.close()
        assert np.array_equal(best, rbest[s]), (k, np.flatnonzero(best != rbest[s])[:8])
        assert n == int((rbest[s] >= 0).sum())
        checked += s.stop - s.start
    assert checked > 0


def test_mixed_batch_equals_single_target_calls(fz):
    c, _ = R.case_and_reference("mixed_batch")
    out = run_device(fz, c)
    for k, t in enumerate(c.targets):
        s = slice(c.q_off[k], c.q_off[k + 1])
        one = run_device(fz, c, [t], np.array([0, s.stop - s.start], np.int32), c.q_lm[s])
        for a, b in zip(out[1:], one[1:]):
            assert np.asarray(a)[s].tobytes() == np.asarray(b).tobytes(), k
