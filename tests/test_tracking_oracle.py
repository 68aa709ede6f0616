"""The tracker's geometry oracle (oracle/tracking_oracle.c: camera::reproject_to_image, frame::can_observe,
landmark::predict_scale_level, the motion model's direction) against the vectorised numpy restatement, bit for bit, on seeded
scenes and at the conventions' knife edges.  CPU only."""
import math

import numpy as np
import pytest

from oracle import tracking as OT
import tracking_problems as TP
import tracking_reference as REF


def _same_bits(a, b):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _check_can_observe(s, usable):
    args = (s["geometry"], s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"], 0.5)
    got = OT.can_observe(*args, usable=usable)
    ref = REF.can_observe(*args, usable=usable)
    for name, a, b in zip(("observable", "reproj_xy", "x_right", "pred_scale_level"), got, ref):
        assert _same_bits(a, b), name
    return got


@pytest.mark.parametrize("name", TP.SCENES)
@pytest.mark.parametrize("masked", [False, True])
def test_can_observe_scenes(name, masked):
    s = TP.scene(name, 4000, seed=11)
    ok, uv, xr, lv = _check_can_observe(s, s["usable"] if masked else None)
    # the scene reaches every outcome: observable, not observable, and more than one level
    assert 0 < ok.sum() < len(ok)
    assert len(np.unique(lv[ok])) >= 3


@pytest.mark.parametrize("name", TP.SCENES)
def test_reproject_scenes(name):
    s = TP.scene(name, 3000, seed=5)
    got = OT.reproject(s["geometry"], s["pos_w"], s["usable"])
    ref = REF.reproject(s["geometry"], s["pos_w"], s["usable"])
    for nm, a, b in zip(("in_image", "reproj_xy", "x_right"), got, ref):
        assert _same_bits(a, b), nm
    if name == "equirectangular":
        assert np.array_equal(got[0], s["usable"].astype(bool))
        assert np.all(got[2][got[0]] == -1.0)


@pytest.mark.parametrize("equirectangular", [False, True])
def test_can_observe_knife_edges(equirectangular):
    s = TP.knife_edges(equirectangular)
    ok, uv, xr, lv = _check_can_observe(s, None)
    if equirectangular:
        return
    P = s["pos_w"]
    # z = 0 and z = -0.0 are behind the camera
    assert not ok[0] and not ok[1] and not ok[2]
    # a reprojection on a bound is inside, one float ulp of x beyond is outside
    for x in (-0.625, 0.625):
        i = np.flatnonzero((P[:, 0] == x) & (P[:, 2] == 1.0))[0]
        assert ok[i] and uv[i, 0] == (0.0 if x < 0 else 640.0)
        beyond = float(np.nextafter(np.float32(x), np.float32(math.copysign(math.inf, x))))
        out = np.flatnonzero((P[:, 0] == beyond) & (P[:, 2] == 1.0))
        assert len(out) and not ok[out].any()
    # the ray cosine: exactly 0.5 passes, a little less fails
    i = np.flatnonzero(P[:, 2] == 2.0)
    i = [k for k in i if s["mean_normal"][k, 0] != 0.0]
    assert ok[i[0]] and not ok[i[1]]
    # NaN and infinite positions are never observable
    assert not ok[~np.isfinite(P).all(1)].any()


def test_scale_range_edges():
    """dist equal to (float)(0.7 min) and (float)(1.3 max) is inside; one float ulp outside is not."""
    s = TP.knife_edges()
    ok = OT.can_observe(s["geometry"], s["pos_w"], s["mean_normal"], s["min_valid_dist"], s["max_valid_dist"])[0]
    onaxis = (s["pos_w"][:, 0] == 0) & (s["pos_w"][:, 1] == 0)
    for mn, mx in ((1.0, 8.0), (0.3, 3.7), (2.0, 2.1)):
        sel = onaxis & (s["min_valid_dist"] == np.float32(mn)) & (s["max_valid_dist"] == np.float32(mx))
        z = s["pos_w"][sel, 2].astype(np.float32)
        lo = np.float32(0.7 * np.float32(mn)); hi = np.float32(1.3 * np.float32(mx))
        for b, inside in ((lo, [False, True, True]), (hi, [True, True, False])):
            k = np.flatnonzero(sel)[np.isin(z, TP._f32_neighbours(b))]
            assert np.array_equal(s["pos_w"][k, 2].astype(np.float32), TP._f32_neighbours(b))
            assert list(ok[k]) == inside


def test_predict_scale_level_edges():
    lsf = np.float32(math.log(2.0))
    # quotients at an integer: ratio 2 and 4 give exactly 1 and 2; one ulp of distance either side moves across the integer
    for d, level in ((4.0, 1), (2.0, 2)):
        q = np.float32(np.float32(math.log(np.float32(8.0) / np.float32(d)))) / lsf
        assert q == level
        for dd in TP._f32_neighbours(d):
            assert OT.predict_scale_level(dd, 8.0, lsf, 8) == int(REF.predict_scale_level(dd, 8.0, lsf, 8)[0])
        assert OT.predict_scale_level(np.nextafter(np.float32(d), np.float32(0)), 8.0, lsf, 8) == level + 1
        assert OT.predict_scale_level(np.nextafter(np.float32(d), np.float32(np.inf)), 8.0, lsf, 8) == level
    # ratio < 1 -> 0, beyond the last level -> clamped, an infinite quotient (distance 0) -> last level, NaN -> 0
    assert OT.predict_scale_level(9.0, 8.0, lsf, 8) == 0
    assert OT.predict_scale_level(0.001, 8.0, lsf, 8) == 7
    assert OT.predict_scale_level(0.0, 8.0, lsf, 8) == 7
    assert OT.predict_scale_level(0.0, 0.0, lsf, 8) == 0
    for d, m in ((9.0, 8.0), (0.001, 8.0), (0.0, 8.0), (0.0, 0.0), (3.0, 8.0)):
        assert OT.predict_scale_level(d, m, lsf, 8) == int(REF.predict_scale_level(d, m, lsf, 8)[0])
    # a sweep of distances through every level of the default pyramid
    d = np.geomspace(0.05, 12.0, 20001).astype(np.float32)
    ref = REF.predict_scale_level(d, 8.0, TP.LOG_SCALE_FACTOR, 8)
    got = np.array([OT.predict_scale_level(x, 8.0, TP.LOG_SCALE_FACTOR, 8) for x in d])
    assert np.array_equal(got, ref)
    assert set(got) == set(range(8))


def test_motion_direction():
    for tb in (0.1, 0.537, 2.0):
        for z, exp in ((tb, (False, False)), (np.nextafter(tb, math.inf), (True, False)), (-tb, (False, False)),
                       (np.nextafter(-tb, -math.inf), (False, True)), (0.0, (False, False))):
            curr = TP.pose12(np.eye(3), [0.0, 0.0, -z])     # trans_wc = (0, 0, z), last frame at the origin: trans_lc.z = z
            last = TP.pose12(np.eye(3), np.zeros(3))
            assert OT.motion_direction(curr, last, False, tb) == exp == REF.motion_direction(curr, last, False, tb)
            assert OT.motion_direction(curr, last, True, tb) == (False, False)
    rng = np.random.default_rng(3)
    for _ in range(200):
        a = TP.pose12(TP.rotation(rng), rng.normal(size=3)); b = TP.pose12(TP.rotation(rng), rng.normal(size=3))
        tb = float(rng.uniform(0.0, 1.0))
        assert OT.motion_direction(a, b, False, tb) == REF.motion_direction(a, b, False, tb)
